"""Host-side checks behind tests/test_gpu_shapes.py: the generalised restatements (oracle/tc_emul.py, oracle/noviews.py) at every
network shape of that file, the skip filter of NeRF.net_params, and the workspace / layout queries against
tests/tc_records.restate_layout."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import noviews as NV, synth, tc_emul as E, torch_ref as T

# id, D, skips, multires, multires_views (None: no view directions), output_ch -- tests/test_gpu_shapes.py's table
SHAPES = [("d2_noenc", 2, [], 0, 0, 5), ("d2_s0", 2, [0], 4, 1, 5), ("d3_s0_v63", 3, [0], 5, 10, 5), ("d4_s4", 4, [4], 10, 4, 5),
          ("d6_s4", 6, [4], 10, 4, 5), ("d7_s2", 7, [2], 8, 4, 5), ("d8_noskip", 8, [], 10, 4, 5), ("d8_s0", 8, [0], 10, 4, 5),
          ("d8_s6", 8, [6], 10, 4, 5), ("nv_d3", 3, [], 6, None, 4), ("nv_d6_s4", 6, [4], 10, None, 5),
          ("nv_d2_s0_noenc", 2, [0], 0, None, 5)]


def _reference_skip(skips, D):
    """the layers after which the reference's NeRF.forward concatenates the input (run_nerf_helpers.py:99-103)"""
    return [i for i in range(D) if i in skips]


@pytest.fixture(scope="module")
def nb():
    import nerf_pytorch_b200
    return nerf_pytorch_b200


def _state(D, skips, L, Lv, out_ch, seed=3):
    ic = E.input_ch(L)
    if Lv is None:
        return NV.nerf_state_noviews(seed, output_ch=out_ch, D=D, input_ch=ic, skips=skips)
    return synth.nerf_state(seed, False, D=D, input_ch=ic, input_ch_views=E.input_ch(Lv), skips=skips)


@pytest.mark.parametrize("sid,D,skips,L,Lv,out_ch", SHAPES, ids=[s[0] for s in SHAPES])
def test_unrounded_emulation_is_the_reference_network(nb, monkeypatch, sid, D, skips, L, Lv, out_ch):
    """With every fp16 rounding switched off, the restated forward is oracle/torch_ref.mlp in float64 and the restated backward
    is float64 autograd of it (the loss scale cancels exactly)."""
    from nerf_pytorch_b200.api import effective_skip
    monkeypatch.setattr(E, "f16", lambda x: x.to(torch.float64))
    monkeypatch.setattr(NV, "f16", lambda x: x.to(torch.float64))
    skip = effective_skip(skips, D)
    assert skip == (_reference_skip(skips, D) or [-1])[0]
    rng = np.random.default_rng(1)
    n_rays, S = 5, 12
    M = n_rays * S
    pts = torch.from_numpy(rng.uniform(-2, 2, (M, 3)).astype(np.float32))
    dirs = rng.standard_normal((n_rays, 3)).astype(np.float32)
    vd = torch.from_numpy(np.repeat(dirs / np.linalg.norm(dirs, axis=-1, keepdims=True), S, 0))
    state = _state(D, skips, L, Lv, out_ch)
    sd = {k: torch.from_numpy(v) for k, v in state.items()}
    ic, views = E.input_ch(L), Lv is not None
    if views:
        em = E.forward(sd, pts, vd, D=D, skip=skip, L=L, Lv=Lv)
    else:
        em = NV.forward_noviews(sd, pts, D=D, skip=skip, L=L)
    assert em["enc64"].shape == (M, 64) and not em["enc64"][:, ic:].any()
    sd_g = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    x = T.embed(pts, L).double()                   # the fp32 encoding both evaluate (as the kernels do)
    if views:
        x = torch.cat([x, T.embed(vd, Lv).double()], -1)
    raw = T.mlp(sd_g, x, ic=ic, icv=E.input_ch(Lv) if views else 0, skip=skip, D=D)
    assert torch.allclose(em["raw"], raw, rtol=1e-12, atol=1e-12), float((em["raw"] - raw).abs().max())
    d_raw = torch.from_numpy(rng.standard_normal((M, 4))) * 1e-3
    (raw * d_raw).sum().backward()
    masks = {"h": [(p > 0).double() for p in em["pre"]]}
    if views:
        masks["hv"] = (em["pre_v"] > 0).double()
        g, _ = E.backward(sd, em, masks, d_raw, 2.0 ** 12, torch.arange(M) // S, n_rays, D=D, skip=skip, L=L)
    else:
        g, _ = NV.backward_noviews(sd, em, masks, d_raw, 2.0 ** 12, D=D, skip=skip, L=L)
    assert set(g) == set(sd_g)
    for name, p in sd_g.items():
        ref = p.grad if p.grad is not None else torch.zeros_like(p)
        err = float((g[name] - ref).norm() / ref.norm().clamp_min(1e-300)) if float(ref.norm()) > 0 else float(g[name].abs().max())
        assert err < 1e-9, (name, err)


def test_default_arguments_are_the_8_layer_net():
    """The defaults are the net every other test uses: 8 layers, skip 4, multires 10 / 4, and the encodings today's formula."""
    rng = np.random.default_rng(2)
    pts = torch.from_numpy(rng.uniform(-2, 2, (40, 3)).astype(np.float32))
    vd = torch.from_numpy(np.repeat(np.array([[0.6, 0.0, 0.8]], np.float32), 40, 0))
    sd = {k: torch.from_numpy(v) for k, v in synth.nerf_state(0).items()}
    a, b = E.forward(sd, pts, vd), E.forward(sd, pts, vd, D=8, skip=4, L=10, Lv=4)
    assert torch.equal(a["enc16"], E.f16(T.embed(pts, 10).double())) and a["enc16"].shape == (40, 63)
    for k in ("enc16", "raw", "hv16", "feat16"):
        assert torch.equal(a[k], b[k]), k
    sdn = {k: torch.from_numpy(v) for k, v in NV.nerf_state_noviews(0).items()}
    assert torch.equal(NV.forward_noviews(sdn, pts)["raw"], NV.forward_noviews(sdn, pts, D=8, skip=4, L=10)["raw"])


@pytest.mark.parametrize("D", range(2, 9))
def test_skip_filter_follows_the_reference(nb, D):
    """net_params' skip is the one entry the reference's loop reaches: entries >= D and negative ones are ignored (create_nerf's
    skips = [4] with netdepth <= 4), entry D - 1 is kept and the library rejects it (the reference fails there), and more
    than one live entry is refused."""
    from nerf_pytorch_b200 import _lib
    from nerf_pytorch_b200.api import effective_skip
    lib = _lib.load()
    for skips in ([], [4], [0], [D - 1], [D - 2], [-1], [D], [D + 3], [4, 9], [-2, 4]):
        live = _reference_skip(skips, D)
        if len(live) > 1:
            with pytest.raises(NotImplementedError):
                effective_skip(skips, D)
            continue
        s = effective_skip(skips, D)
        assert s == (live[0] if live else -1), (skips, D)
        n = _lib.NerfNetParams(D=D, W=256, input_ch=63, input_ch_views=27, skip=s, use_viewdirs=1, output_ch=4)
        accepted = lib.nerf_b200_packed_bytes(C.byref(n)) > 0
        assert accepted == (s < D - 1), (skips, D, lib.nerf_b200_last_error())
    with pytest.raises(NotImplementedError):
        effective_skip([0, 1], D)


def _sms(lib, n):
    """the SM count the library plans with (132 without a device): the grid of a batch with more super-tiles than SMs"""
    out = (C.c_int64 * 12)()
    assert lib.nerf_b200_march_bwd_tc_layout(1 << 20, 256, C.byref(n), out) == 0
    return int(out[5])


@pytest.mark.parametrize("sid,D,skips,L,Lv,out_ch", SHAPES, ids=[s[0] for s in SHAPES])
def test_layout_queries_match_the_restatement(nb, sid, D, skips, L, Lv, out_ch):
    import tc_records as R
    from nerf_pytorch_b200 import _lib
    from nerf_pytorch_b200.api import effective_skip
    lib = _lib.load()
    icv = E.input_ch(Lv) if Lv is not None else 0
    n = _lib.NerfNetParams(D=D, W=256, input_ch=E.input_ch(L), input_ch_views=icv, skip=effective_skip(skips, D),
                           use_viewdirs=int(Lv is not None), output_ch=out_ch)
    sms = _sms(lib, n)
    for N, S in ((37, 70), (1, 1), (7, 1), (50, 2), (20, 129), (sms, 256), (5, 300), (5, 1024), (4 * sms, 128), (4096, 192)):
        layout, ws, rec = R.restate_layout(N, S, D, icv, sms)
        out = (C.c_int64 * 12)()
        assert lib.nerf_b200_march_bwd_tc_layout(N, S, C.byref(n), out) == 0, lib.nerf_b200_last_error()
        assert tuple(int(v) for v in out) == layout, (N, S)
        assert lib.nerf_b200_march_bwd_tc_workspace_bytes(N, S, C.byref(n)) == ws, (N, S)
        ab, mb = C.c_size_t(0), C.c_size_t(0)
        assert lib.nerf_b200_train_record_bytes(N, S, C.byref(n), C.byref(ab), C.byref(mb)) == 0
        assert (ab.value, mb.value) == rec, (N, S)
