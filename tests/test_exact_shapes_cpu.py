"""Host-side checks behind section (e) of tests/test_gpu_shapes.py: networks only the exact path (fp32 CUDA cores) serves.

  * a float64 restatement of render() + img2mse + autograd (oracle/torch_ref.mlp / composite, oracle/resample.fine_z) reproduces
    the reference's own results in tests/golden/exact_shapes.npz (oracle/gen_shapes_golden.py): this pins the fixture and the
    restatement the GPU tests use;
  * the library refuses a skip after the last layer, a width that is not a multiple of 4 or above 256, and a depth above
    NERF_B200_MAX_D on every exact entry point during argument validation (nothing is launched or dereferenced), with messages
    naming the rule; NeRF.net_params() refuses netdepth > 16 the same way;
  * the reference's network itself fails with a skip after the last layer;
  * the tensor-core path's refusal of another width points to the exact path.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2
from oracle import nerf_oracle as O
from oracle import noviews, resample, synth, tc_emul
from oracle import torch_ref as T

EXACT_GOLDEN_CASES = ["w128_d10", "L14_Lv8", "w100_nv_odd"]


def _states(fx, p):
    views = bool(fx[p + "use_viewdirs"])
    ic = tc_emul.input_ch(int(fx[p + "multires"]))
    icv = tc_emul.input_ch(int(fx[p + "multires_views"])) if views else 0
    out = []
    for k, tag in enumerate(("", "_fine")):
        D, W = int(fx[p + "netdepth" + tag]), int(fx[p + "netwidth" + tag]) if p + "netwidth" + tag in fx else 256
        seed = int(fx[p + "seed_w"]) + k
        if views:
            out.append((D, synth.nerf_state(seed, False, D=D, W=W, input_ch=ic, input_ch_views=icv, skips=(4,))))
        else:
            out.append((D, noviews.nerf_state_noviews(seed, output_ch=int(fx[p + "output_ch"]), D=D, W=W, input_ch=ic, skips=(4,))))
    return ic, icv, out


def _restated_render(fx, case, dtype=torch.float64):
    """render() of one fixture case on the fp32 ray batch the kernels read, in float64 (or float32: how far fp32 arithmetic
    itself is from it) -> (loss, maps, grads of the coarse and fine net by parameter name)"""
    p = case + "_"
    views = bool(fx[p + "use_viewdirs"])
    L, Lv = int(fx[p + "multires"]), int(fx[p + "multires_views"])
    ic, icv, nets = _states(fx, p)
    rays = fx[p + "rays"]
    packed = O.pack_rays(int(fx[p + "H"]), int(fx[p + "W"]), fx[p + "K"], rays[0], rays[1], bool(fx[p + "ndc"]),
                         float(fx[p + "near"]), float(fx[p + "far"]), views).astype(np.float64 if dtype == torch.float64 else np.float32)
    white = bool(fx[p + "white_bkgd"])
    Sc, Ni = int(fx[p + "N_samples"]), int(fx[p + "N_importance"])
    o, d = torch.from_numpy(packed[:, 0:3]), torch.from_numpy(packed[:, 3:6])
    npt = packed.dtype
    sds = [{k: torch.from_numpy(v).to(dtype).requires_grad_(True) for k, v in st.items()} for _, st in nets]

    def net_pass(sd, D, z):
        N, S = z.shape
        x = T.embed((o[:, None] + d[:, None] * torch.from_numpy(z)[..., None]).reshape(-1, 3), L)
        if views:
            x = torch.cat([x, T.embed(torch.from_numpy(np.repeat(packed[:, 8:11], S, 0)), Lv)], -1)
        raw = T.mlp(sd, x, ic=ic, icv=icv, skip=4 if D > 4 else -1, D=D)        # create_nerf: skips = [4]
        return T.composite(raw.reshape(N, S, 4), torch.from_numpy(z), d, white)

    z_c = resample.coarse_z(packed[:, 6:7], packed[:, 7:8], Sc, dtype=npt)
    rgb0, _, _, w0 = net_pass(sds[0], nets[0][0], z_c)
    z_f, _, _ = resample.fine_z(z_c, w0.detach().numpy(), Ni, det=True, dtype=npt)
    rgb, disp, acc, _ = net_pass(sds[1], nets[1][0], z_f)
    target = torch.from_numpy(fx[p + "target"]).to(dtype)
    loss = ((rgb - target) ** 2).mean() + ((rgb0 - target) ** 2).mean()
    loss.backward()
    grads = [{k: (v.grad if v.grad is not None else torch.zeros_like(v)).numpy().reshape(-1) for k, v in sd.items()} for sd in sds]
    maps = {"rgb_map": rgb.detach().numpy(), "disp_map": disp.detach().numpy(), "acc_map": acc.detach().numpy()}
    return float(loss.detach()), maps, grads


@pytest.mark.parametrize("case", EXACT_GOLDEN_CASES)
def test_restatement_reproduces_the_reference(case):
    """The fixture's reference ran in fp32: the float64 restatement is within 2e-5 plus twice the restatement's own fp32
    distance of its maps and loss, and its gradients within 1e-5 plus twice the distance of the reference's own float64 run
    (g_{c,f}_cond).  The restatement starts from the fp32 ray batch, the float64 reference from float64 rays: at 2^13 the
    encoding turns that rounding into phase, so the two float64 runs are not the same."""
    fx = load_golden("exact_shapes")
    p = case + "_"
    assert int(fx[p + "N_importance"]) > 0
    loss, maps, grads = _restated_render(fx, case)
    loss32, maps32, _ = _restated_render(fx, case, torch.float32)
    assert abs(loss - float(fx[p + "loss"])) <= 2e-5 * loss + 2 * abs(loss32 - loss), (loss, loss32, float(fx[p + "loss"]))
    for k, v in maps.items():
        ref = fx[p + k].astype(np.float64)
        assert np.array_equal(np.isnan(v), np.isnan(ref)) and np.array_equal(np.isnan(v), np.isnan(maps32[k])), k
        ok = ~np.isnan(ref)
        e, cond = rel_l2(v[ok], ref[ok]), rel_l2(maps32[k][ok], v[ok])
        assert e <= 2e-5 + 2 * cond, (k, e, cond)
    for tag, g in zip(("c", "f"), grads):
        names = [str(s) for s in fx[f"{p}g_{tag}_names"]]
        assert names == list(g), (names, list(g))
        ends = np.cumsum(fx[f"{p}g_{tag}_count"])
        for j, name in enumerate(names):
            sl = slice(ends[j - 1] if j else 0, ends[j])
            idx, ref, cond = fx[f"{p}g_{tag}_idx"][sl], fx[f"{p}g_{tag}_val"][sl].astype(np.float64), float(fx[f"{p}g_{tag}_cond"][j])
            if float(fx[f"{p}g_{tag}_norm"][j]) == 0.0:           # not on the loss's graph
                assert not g[name].any(), (tag, name)
                continue
            err = float(np.linalg.norm(g[name][idx] - ref) / max(np.linalg.norm(ref), 1e-30))
            assert err <= 1e-5 + 2 * cond, (tag, name, err, cond)


# ---- refusals ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from nerf_pytorch_b200 import _lib
    return _lib


# id -> (NerfNetParams fields, what the message names)
REFUSED = {
    "skip_D_minus_1": (dict(D=4, W=128, skip=3), "skip layer must be < netdepth - 1"),
    "W50": (dict(D=8, W=50, skip=4), "netwidth <= 256 and a multiple of 4"),
    "W260": (dict(D=8, W=260, skip=4), "netwidth <= 256 and a multiple of 4"),
    "D17": (dict(D=17, W=128, skip=4), "1 <= netdepth <= 16"),
}


@pytest.mark.parametrize("views", [True, False], ids=["views", "noviews"])
@pytest.mark.parametrize("case", list(REFUSED))
def test_exact_path_refuses_during_argument_validation(lib, case, views):
    """Every exact entry point refuses the net before it launches or dereferences anything: the pointers are fake."""
    fields, msg = REFUSED[case]
    L = lib.load()
    n = lib.NerfNetParams(input_ch=63, input_ch_views=27 if views else 0, use_viewdirs=int(views), output_ch=4 if views else 5, **fields)
    cfg = lib.NerfRenderCfg(N_samples=16, N_importance=16, multires=10, multires_views=4, ray_stride=11 if views else 8,
                            precision=lib.PREC_FP32)
    fake = C.c_void_p(256)
    out = lib.NerfPassOut(fake, fake, fake, fake, fake, fake)
    gr = lib.NerfNetGrads()
    launches = L.nerf_b200_launch_count()

    def refused(rc):
        err = L.nerf_b200_last_error().decode()
        return rc != 0 and msg in err, err
    calls = {
        "march": lambda: L.nerf_b200_march(fake, fake, None, 8, 16, C.byref(n), None, C.byref(cfg), C.byref(out), fake, 1 << 30, None),
        "run_network": lambda: L.nerf_b200_run_network(fake, fake, 8, 16, C.byref(n), None, 10, 4, lib.PREC_FP32, fake, fake, 1 << 30, None),
        "march_bwd": lambda: L.nerf_b200_march_bwd(fake, fake, None, 8, 16, C.byref(n), None, C.byref(cfg), fake, C.byref(gr),
                                                   fake, 1 << 30, None),
        "march_bwd_outs": lambda: L.nerf_b200_march_bwd_outs(fake, fake, None, 8, 16, C.byref(n), None, C.byref(cfg),
                                                             C.byref(lib.NerfOutGrads(rgb_map=fake)), C.byref(gr), fake, 1 << 30, None),
        "render_rays_fwd": lambda: L.nerf_b200_render_rays_fwd(fake, 8, C.byref(cfg), C.byref(n), None, C.byref(n), None, fake, fake,
                                                               None, None, None, None, fake, C.byref(out), fake, fake, C.byref(out),
                                                               fake, 1 << 30, None),
    }
    for name, call in calls.items():
        ok, err = refused(call())
        assert ok, (name, err)
    assert L.nerf_b200_march_bwd_workspace_bytes(8, 16, C.byref(n)) == 0
    assert msg in L.nerf_b200_last_error().decode()
    assert L.nerf_b200_launch_count() == launches


def test_exact_path_accepts_its_shapes(lib):
    """The limits themselves are accepted: width 4 and 256, depth 1 and 16, skip D - 2."""
    L = lib.load()
    for D, W, skip in ((1, 4, -1), (16, 256, 14), (2, 36, -1), (9, 252, 7), (16, 64, 0)):
        n = lib.NerfNetParams(D=D, W=W, skip=skip, input_ch=99, input_ch_views=99, use_viewdirs=1, output_ch=4)
        assert L.nerf_b200_march_bwd_workspace_bytes(8, 16, C.byref(n)) > 0, (D, W, skip, L.nerf_b200_last_error())


def test_net_params_refuses_netdepth_above_16():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib
    net = nb.NeRF(D=_lib.MAX_D + 1, W=8, input_ch=3, input_ch_views=3, output_ch=4, skips=[], use_viewdirs=False)
    with pytest.raises(RuntimeError, match="netdepth must be in \\[1, 16\\]"):
        net.net_params()


def test_reference_network_fails_on_a_skip_after_the_last_layer():
    """The reference's heads take W columns; a skip after the last layer hands them W + input_ch."""
    D, ic, icv = 4, 63, 27
    sd = {k: torch.from_numpy(v).double() for k, v in synth.nerf_state(0, D=D, W=32, input_ch=ic, input_ch_views=icv, skips=(2,)).items()}
    x = torch.zeros(5, ic + icv, dtype=torch.float64)
    T.mlp(sd, x, ic=ic, icv=icv, skip=2, D=D)              # D - 2: a net the library runs
    with pytest.raises(RuntimeError):
        T.mlp(sd, x, ic=ic, icv=icv, skip=D - 1, D=D)


def test_tensor_core_refusal_points_to_the_exact_path(lib):
    L = lib.load()
    n = lib.NerfNetParams(D=8, W=128, skip=4, input_ch=63, input_ch_views=27, use_viewdirs=1, output_ch=4)
    assert L.nerf_b200_packed_bytes(C.byref(n)) == 0
    err = L.nerf_b200_last_error().decode()
    assert "netwidth == 256" in err and "set_precision('fp32')" in err, err
