"""set_backward('tc_split'): training at fp32 fidelity on tensor cores.  Under precision tc_split, a call that needs gradients runs
the split training forward (march_split_train_kernel: hi + lo tile records) and the split backward (dgrad_split_kernel, the
split seed kernels, the weight gradient as dA_hi^T H_hi + dA_lo^T H_hi + dA_hi^T H_lo).

(a) the split training image starts with packed_split()'s bytes, and the training-mode forward returns the inference pass's bits;
(b) gradients on trained_lego_grads against the reference's autograd and against the exact recompute backward on the same split
    forward, >= 20x closer to the latter than the tc_fp16 backward is; the same for a loss on every output and a net without
    view directions;
(c) run-to-run bits, and the refusal under the other precisions before any launch.
Measured deviations go to parity_split_backward.json in $NERF_B200_PARITY_DIR (default: a nerf_b200_parity directory under the
system's temporary directory)."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from conftest import load_golden
from test_gpu_parity import _trained_nets

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


@pytest.fixture
def modes(G):
    yield
    G.nb.set_precision("tc_fp16")
    G.nb.set_backward("tc")


def _record(name, value):
    out_dir = os.environ.get("NERF_B200_PARITY_DIR") or os.path.join(tempfile.gettempdir(), "nerf_b200_parity")
    path = os.path.join(out_dir, "parity_split_backward.json")
    os.makedirs(out_dir, exist_ok=True)
    data = {}
    if os.path.isfile(path):
        with open(path) as f:
            data = json.load(f)
    data[name] = value
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def _lego(G, fx):
    return G.synth.ray_batch("lego", int(fx["N"]), seed=int(fx["ray_seed"]))


def _render(G, nets, sb, retraw=False, use_viewdirs=True, N_importance=128):
    return G.nb.render(sb["H"], sb["W"], sb["K"], chunk=32768, rays=G.dev(sb["rays"]), ndc=False, near=2., far=6.,
                       use_viewdirs=use_viewdirs, network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(),
                       N_samples=64, N_importance=N_importance, perturb=0., white_bkgd=True, raw_noise_std=0., retraw=retraw)


def _loss(G, out, target, kind):
    rgb, disp, acc, ex = out
    loss = G.nb.img2mse(rgb, target) + G.nb.img2mse(ex["rgb0"], target)
    if kind == "all":
        finite = torch.isfinite(disp)                # disp is NaN on rays with acc = 0, as in the reference
        loss = loss + ((acc - 0.5) ** 2).mean() + 0.1 * ((disp[finite] - 0.3) ** 2).mean() + 1e-3 * (ex["raw"] ** 2).mean()
    return loss


def _grads(G, nets, sb, target, precision, backward, kind="rgb", use_viewdirs=True):
    G.nb.set_precision(precision)
    G.nb.set_backward(backward)
    for n in nets:
        n.zero_grad(set_to_none=True)
    loss = _loss(G, _render(G, nets, sb, retraw=True, use_viewdirs=use_viewdirs), target, kind)
    loss.backward()
    torch.cuda.synchronize()
    return {f"{t}.{k}": p.grad.detach().clone() for t, n in zip("cf", nets) for k, p in n.named_parameters()}, float(loss)


def _rel(a, b):
    return float(torch.linalg.norm((a - b).double()) / max(float(torch.linalg.norm(b.double())), 1e-30))


def _median_rel(ga, gb):
    return float(np.median([_rel(ga[k], gb[k]) for k in gb]))


def _check_backward_stream(img, off, net):
    """The split training image's backward stream restated in numpy: chunk c holds W^T[32 c .. 32 c + 31] of its layer (views_linears[0]
    [:, :W], feature_linear, pts_linears[D-1 .. 1] over their h columns) scaled by the layer's power of two (largest |w| into
    [2^13, 2^14)), as two 16 KB stages of 16 columns, each row [8 hi | 8 hi | 8 lo | 8 lo] fp16 in SWIZZLE_64B order; hi is
    fp16(w s) and hi + lo rebuilds w s to fp16's 22 significant bits."""
    P = {k: v.detach().cpu().numpy().astype(np.float32) for k, v in net.named_parameters()}
    D, IC = 8, 63

    def scale(w):
        _, e = np.frexp(np.abs(w).max())
        return np.float32(2.0 ** (14 - int(e)))
    layers = [(P["views_linears.0.weight"][:, :256], P["views_linears.0.weight"][:, :256], 4),
              (P["feature_linear.weight"], P["feature_linear.weight"], 8)]
    for l in range(D - 1, 0, -1):
        w = P[f"pts_linears.{l}.weight"]
        layers.append((w[:, IC:] if l == 5 else w, w, 8))
    row = np.arange(256)[:, None]
    col = np.arange(16)[None, :]
    for h_w, full, nch in layers:
        s = scale(full)
        wt = (h_w * s).astype(np.float32)                       # chunk element (row n, column k) = wt[32 c + k][n]
        for c in range(nch):
            for h in range(2):
                k = 32 * c + 16 * h + col                        # W^T row (input column of the layer)
                want = np.where(k < wt.shape[0], wt[np.minimum(k, wt.shape[0] - 1), row], 0).astype(np.float32)
                unit = (col // 8)
                base = off + h * 256 * 64 + (row >> 3) * 512 + (row & 7) * 64 + (col % 8) * 2
                hi_at = base + ((unit ^ ((row & 7) >> 1)) << 4)
                lo_at = base + (((unit + 2) ^ ((row & 7) >> 1)) << 4)
                hi = img.view(np.uint8)[np.stack([hi_at, hi_at + 1], -1)].copy().view(np.float16)[..., 0].astype(np.float32)
                lo = img.view(np.uint8)[np.stack([lo_at, lo_at + 1], -1)].copy().view(np.float16)[..., 0].astype(np.float32)
                assert np.array_equal(hi, want.astype(np.float16).astype(np.float32))
                assert np.all(np.abs(hi + lo - want) <= np.abs(want) * 2.0 ** -21 + 2.0 ** -24)
            off += 2 * 256 * 64
    assert off == img.size                                   # the stream ends the image


# ---- (a) image and forward -----------------------------------------------------------------------------------------------------

def test_split_train_image_and_forward_bits(G, modes):
    import ctypes as C
    lib = G._lib.load()
    nets = _trained_nets(G)
    for n in nets:                                  # both packed into zeroed buffers: the bytes no kernel writes compare equal too
        p = n.net_params()
        na, nb_ = lib.nerf_b200_packed_bytes_split(C.byref(p)), lib.nerf_b200_packed_bytes_split_train(C.byref(p))
        assert nb_ > na
        a, b = torch.zeros(na, dtype=torch.uint8, device=G.DEV), torch.zeros(nb_, dtype=torch.uint8, device=G.DEV)
        assert lib.nerf_b200_pack_weights_split(C.byref(p), G.ptr(a), na, G.stream()) == 0
        assert lib.nerf_b200_pack_weights_split_train(C.byref(p), G.ptr(b), nb_, G.stream()) == 0
        assert torch.equal(b[:na], a)
        _check_backward_stream(b.cpu().numpy(), (na + 1023) // 1024 * 1024, n)
    fx = load_golden("trained_lego_grads")
    sb = _lego(G, fx)
    G.nb.set_precision("tc_split")
    with torch.no_grad():
        ref = _render(G, nets, sb, retraw=True)
    G.nb.set_backward("tc_split")
    got = _render(G, nets, sb, retraw=True)
    assert got[0].grad_fn is not None
    for a, b in ((ref[0], got[0]), (ref[1], got[1]), (ref[2], got[2]), (ref[3]["rgb0"], got[3]["rgb0"]), (ref[3]["raw"], got[3]["raw"])):
        assert torch.equal(a.detach().contiguous().view(torch.int32), b.detach().contiguous().view(torch.int32))


# ---- (b) gradients -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["rgb", "all"])
def test_trained_gradients_against_exact_and_reference(G, modes, kind):
    fx = load_golden("trained_lego_grads")
    sb = _lego(G, fx)
    nets = _trained_nets(G)
    target = G.dev(fx["target"])
    g_split, l_split = _grads(G, nets, sb, target, "tc_split", "tc_split", kind)
    g_exact, l_exact = _grads(G, nets, sb, target, "tc_split", "exact", kind)
    g_fp16, _ = _grads(G, nets, sb, target, "tc_fp16", "tc", kind)
    st = {"split_vs_exact_median": _median_rel(g_split, g_exact),
          "split_vs_exact_max": max(_rel(g_split[k], g_exact[k]) for k in g_exact),
          "fp16_vs_exact_median": _median_rel(g_fp16, g_exact),
          "loss_split_vs_exact": abs(l_split - l_exact) / l_exact,
          "per_tensor": {k: _rel(g_split[k], g_exact[k]) for k in g_exact}}
    if kind == "rgb":
        errs = []
        for tag, net in zip("cf", nets):
            for name, _ in net.named_parameters():
                g = g_split[f"{tag}.{name}"].cpu().numpy().reshape(-1)
                idx, ref = fx[f"g_{tag}_{name}_idx"], fx[f"g_{tag}_{name}_val"]
                errs.append(float(np.linalg.norm(g[idx] - ref) / max(np.linalg.norm(ref), 1e-12)))
        st["split_vs_reference_median"], st["split_vs_reference_max"] = float(np.median(errs)), float(max(errs))
    _record(f"trained_grads_{kind}", st)
    print(kind, st)
    assert l_split == l_exact                       # the same split forward
    # gates ~3x the values measured on an H100 (median 3.2e-5 / 2.4e-5, max 9.8e-4; against the reference 5.9e-5 / 5.4e-3)
    assert st["split_vs_exact_median"] * 20 <= st["fp16_vs_exact_median"], st
    assert st["split_vs_exact_median"] < 1e-4 and st["split_vs_exact_max"] < 3e-3, st
    # per tensor: 3x the value measured on an H100 (floor 1e-6).  A lo term dropped anywhere moves its tensors by ~1e-4 or more,
    # which the tensors read by one kernel only (alpha_linear, the view columns, rgb_linear: ~3e-6 measured) exceed many times
    with open(os.path.join(os.path.dirname(__file__), "golden", "split_backward_gates.json")) as f:
        gates = json.load(f)[kind]
    over = {k: (v, gates[k]) for k, v in st["per_tensor"].items() if not v <= gates[k]}
    assert not over, over
    if kind == "rgb":
        assert st["split_vs_reference_median"] < 2e-4 and st["split_vs_reference_max"] < 1.6e-2, st


def test_noviews_gradients_against_exact(G, modes):
    """a default-initialised net without view directions (output_linear head, the split dA_{D-1} seed), coarse pass only"""
    torch.manual_seed(0)
    net = G.nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=0, output_ch=5, skips=[4], use_viewdirs=False).to(G.DEV)
    fx = load_golden("trained_lego_grads")
    sb = _lego(G, fx)
    target = G.dev(fx["target"])

    def grads(precision, backward):
        G.nb.set_precision(precision)
        G.nb.set_backward(backward)
        net.zero_grad(set_to_none=True)
        rgb, _, _, _ = _render(G, (net, None), sb, use_viewdirs=False, N_importance=0)
        G.nb.img2mse(rgb, target).backward()
        return {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}

    g_split, g_exact, g_fp16 = grads("tc_split", "tc_split"), grads("tc_split", "exact"), grads("tc_fp16", "tc")
    st = {"split_vs_exact_median": _median_rel(g_split, g_exact), "fp16_vs_exact_median": _median_rel(g_fp16, g_exact)}
    _record("noviews_grads", st)
    print(st)
    assert set(g_split) == set(g_exact)
    assert st["split_vs_exact_median"] * 20 <= st["fp16_vs_exact_median"], st
    assert st["split_vs_exact_median"] < 1e-5, st                 # measured 2.9e-6 on an H100


# ---- (c) plumbing --------------------------------------------------------------------------------------------------------------

def test_run_to_run_bits(G, modes):
    fx = load_golden("trained_lego_grads")
    sb = _lego(G, fx)
    nets = _trained_nets(G)
    target = G.dev(fx["target"])
    a, _ = _grads(G, nets, sb, target, "tc_split", "tc_split", "all")
    b, _ = _grads(G, nets, sb, target, "tc_split", "tc_split", "all")
    for k in a:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k


@pytest.mark.parametrize("precision", ["tc_fp16", "fp32"])
def test_split_backward_is_refused_in_other_precisions(G, modes, precision):
    fx = load_golden("trained_lego_grads")
    sb = _lego(G, fx)
    nets = _trained_nets(G)
    G.nb.set_precision(precision)
    G.nb.set_backward("tc_split")
    n0 = G.nb.launch_count()
    with pytest.raises(RuntimeError, match="tc_split"):
        _render(G, nets, sb)
    assert G.nb.launch_count() == n0
    with torch.no_grad():                           # inference is unaffected
        _render(G, nets, sb)
    assert G.nb.launch_count() > n0
