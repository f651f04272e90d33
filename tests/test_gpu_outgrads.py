"""Losses on disp_map, acc_map and raw (not only rgb_map) through both backward paths, on the GPU.

  1. raw2outputs(): the gradient of each output alone and of their sum against the float64 restatement (oracle/outgrads.py);
     with only rgb seeded the _outs entry point is bitwise the rgb-only one;
  2. render(): disp, acc, disp0, acc0 and raw carry a gradient, and mean(acc).backward() alone works;
  3. exact backward against the reference's autograd (tests/golden/outgrads.npz), every case and loss;
  4. tensor-core pass, stage check: dL/draw and the loss-scale input read from the workspace against the restatement;
  5. tensor-core against exact backward on the same fp16 forward, every case and loss and the render options;
  6. 4096 rays: three tensor-core evaluations of L_all agree.
Measured deviations go to parity_outgrads.json in $NERF_B200_PARITY_DIR (default: a nerf_b200_parity directory under the
system's temporary directory)."""
import ctypes as C
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden, rel_l2
from oracle import outgrads as OG
from oracle import tc_emul

pytestmark = pytest.mark.gpu

CASES = ("a", "b", "c")


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


@pytest.fixture(scope="module")
def FX():
    return load_golden("outgrads")


def _record(name, value):
    out_dir = os.environ.get("NERF_B200_PARITY_DIR") or os.path.join(tempfile.gettempdir(), "nerf_b200_parity")
    path = os.path.join(out_dir, "parity_outgrads.json")
    os.makedirs(out_dir, exist_ok=True)
    data = {}
    if os.path.isfile(path):
        with open(path) as f:
            data = json.load(f)
    data[name] = value
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


class _Spy:
    """counts the calls of some C entry points (forwarded unchanged)"""

    def __init__(self, monkeypatch, lib, names):
        self.calls = {n: 0 for n in names}
        for n in names:
            fn = getattr(lib, n)

            def wrap(*a, _fn=fn, _n=n):
                self.calls[_n] += 1
                return _fn(*a)
            monkeypatch.setattr(lib, n, wrap)


# ---- 1. raw2outputs ---------------------------------------------------------------------------------------------------

def _r2o_problem(seed, N=64, S=96):
    rng = np.random.default_rng(seed)
    raw = (rng.standard_normal((N, S, 4)) * 2).astype(np.float32)
    z = np.sort(rng.random((N, S), dtype=np.float32) * 4 + 2, -1)
    d = rng.standard_normal((N, 3)).astype(np.float32)
    seeds = dict(rgb_map=rng.standard_normal((N, 3)), disp_map=rng.standard_normal(N), acc_map=rng.standard_normal(N),
                 depth_map=rng.standard_normal(N), weights=rng.standard_normal((N, S)))
    return raw, z, d, {k: v.astype(np.float32) for k, v in seeds.items()}


R2O_OUTS = ("rgb_map", "disp_map", "acc_map", "weights", "depth_map")       # raw2outputs' return order


@pytest.mark.parametrize("white_bkgd", [False, True])
@pytest.mark.parametrize("which", list(R2O_OUTS) + ["sum"])
def test_raw2outputs_output_gradients(G, white_bkgd, which):
    raw, z, d, seeds = _r2o_problem(1)
    r = G.dev(raw).requires_grad_(True)
    outs = dict(zip(R2O_OUTS, G.nb.raw2outputs(r, G.dev(z), G.dev(d), 0., white_bkgd)))
    keys = R2O_OUTS if which == "sum" else (which,)
    loss = sum((outs[k] * G.dev(seeds[k])).sum() for k in keys)
    loss.backward()
    ref = OG.adjoint(torch.from_numpy(raw), torch.from_numpy(z), torch.from_numpy(d), white_bkgd,
                     {k: torch.from_numpy(seeds[k]) for k in keys}).numpy()
    err = rel_l2(r.grad.cpu().numpy(), ref)
    _record(f"raw2outputs_{which}_wb{int(white_bkgd)}", err)
    assert err < 2e-5, (which, err)


def test_raw2outputs_rgb_only_outs_is_bitwise_the_rgb_entry(G):
    raw, z, d, seeds = _r2o_problem(2)
    lib = G._lib.load()
    N, S = z.shape
    r, zz, dd, g = G.dev(raw), G.dev(z), G.dev(d), G.dev(seeds["rgb_map"])
    noise = G.dev((np.random.default_rng(3).random((N, S)) * 0.5).astype(np.float32))
    for nz in (None, noise):
        a, b = torch.empty_like(r), torch.empty_like(r)
        G._lib.check(lib.nerf_b200_raw2outputs_bwd(G.ptr(r), G.ptr(zz), G.ptr(dd), 3, G.ptr(nz), N, S, 1, G.ptr(g), G.ptr(a), G.stream()), "bwd")
        og = G._lib.NerfOutGrads(rgb_map=G.ptr(g))
        G._lib.check(lib.nerf_b200_raw2outputs_bwd_outs(G.ptr(r), G.ptr(zz), G.ptr(dd), 3, G.ptr(nz), N, S, 1, C.byref(og), G.ptr(b),
                                                        G.stream()), "bwd_outs")
        torch.cuda.synchronize()
        assert torch.equal(a, b)


# ---- 2. render(): differentiable outputs ------------------------------------------------------------------------------

def test_render_outputs_carry_gradients(G):
    sb = G.synth.ray_batch("lego", 32, seed=12)
    nets = _nets(G, "a")
    rgb, disp, acc, ex = G.nb.render(400, 400, sb["K"], rays=G.dev(sb["rays"]), ndc=False, near=2., far=6., use_viewdirs=True,
                                     network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64,
                                     N_importance=64, perturb=0., white_bkgd=True, raw_noise_std=0., retraw=True)
    for t in (rgb, disp, acc, ex["rgb0"], ex["disp0"], ex["acc0"], ex["raw"]):
        assert t.requires_grad
    assert not ex["z_std"].requires_grad
    torch.mean(acc).backward()
    g = nets[1].pts_linears[0].weight.grad
    assert g is not None and bool(torch.isfinite(g).all()) and float(g.abs().max()) > 0
    # acc alone reaches the fine net only: the coarse net's gradient is zero
    assert float(nets[0].pts_linears[0].weight.grad.abs().max()) == 0.0


# ---- fixture cases ----------------------------------------------------------------------------------------------------

def _trained():
    return OG.trained_states(os.path.join(GOLDEN, "trained_weights.npz"))


def _nets(G, case):
    """a and c: the trained nets; b: a net without view directions with their density (oracle/outgrads.noviews_from_trained)"""
    tr = _trained()
    if case == "b":
        return [G.make_net(OG.noviews_from_trained(tr[k], k), use_viewdirs=False) for k in (0, 1)]
    return [G.make_net(s) for s in tr]


def _opts(case):
    return dict(N_importance=64 if case == "c" else 128, perturb=1. if case == "c" else 0., raw_noise_std=1. if case == "c" else 0.,
                pytest=case == "c", use_viewdirs=case != "b")


def _render_case(G, fx, case, loss_name, prec, bwd, nets=None, **over):
    nets = nets if nets is not None else _nets(G, case)
    o = _opts(case)
    o.update(over)
    G.nb.set_precision(prec)
    G.nb.set_backward(bwd)
    try:
        rgb, disp, acc, ex = G.nb.render(int(fx[f"{case}_H"]), int(fx[f"{case}_W"]), fx[f"{case}_K"], chunk=32768,
                                         rays=G.dev(fx[f"{case}_rays"]), ndc=bool(fx[f"{case}_ndc"]), near=float(fx[f"{case}_near"]),
                                         far=float(fx[f"{case}_far"]), network_fn=nets[0], network_fine=nets[1],
                                         network_query_fn=G.query_fn(), N_samples=64, white_bkgd=bool(fx[f"{case}_white_bkgd"]),
                                         retraw=True, **o)
        if o["N_importance"] == 0:
            ex = dict(ex, rgb0=rgb, disp0=disp, acc0=acc)
        loss = OG.loss_of(loss_name, rgb, disp, acc, ex, G.dev(fx[f"{case}_target"]), G.dev(fx[f"{case}_t_acc"]))
        loss.backward()
    finally:
        G.nb.set_precision("tc_fp16")
        G.nb.set_backward("tc")
    torch.cuda.synchronize()
    return float(loss.item()), nets


def _grads(nets):
    return {(k, name): p.grad.detach().double().cpu() for k, n in enumerate(nets) if n is not None for name, p in n.named_parameters()
            if p.grad is not None}


# ---- 3. exact backward vs the reference's autograd ----------------------------------------------------------------------

@pytest.mark.parametrize("loss_name", OG.LOSSES)
@pytest.mark.parametrize("case", CASES)
def test_exact_backward_matches_reference(G, FX, case, loss_name):
    loss, nets = _render_case(G, FX, case, loss_name, "fp32", "exact")
    ref_loss = float(FX[f"{case}_{loss_name}_loss"])
    if np.isnan(ref_loss):                     # a ray with acc = 0: the reference's disp is NaN there, and so is its mean
        assert np.isnan(loss)
    else:
        # L_raw averages the trained net's raw sigma (up to ~1e3 at surfaces), which moves with the fine samples' positions:
        # 1e-4 there, 1e-5 for the composited losses
        tol = 1e-4 if loss_name == "raw" else 1e-5
        assert abs(loss - ref_loss) <= tol * abs(ref_loss), (loss, ref_loss)
    errs = {}
    for tag, net in (("c", nets[0]), ("f", nets[1])):
        names = [str(s) for s in FX[f"{case}_g_{tag}_names"]]
        assert names == [n for n, _ in net.named_parameters()]
        ends = np.cumsum(FX[f"{case}_g_{tag}_count"])
        idx_all = FX[f"{case}_g_{tag}_idx"]
        val_all, norm_all, on_all, cond_all = (FX[f"{case}_{loss_name}_g_{tag}_{k}"] for k in ("val", "norm", "on", "cond"))
        for j, (name, p) in enumerate(net.named_parameters()):
            key = f"{case}_{loss_name}_g_{tag}_{name}"
            g = p.grad.detach().cpu().numpy().reshape(-1)
            if not on_all[j]:                  # not on the loss's graph in the reference
                assert not g.any(), key
                continue
            sl = slice(ends[j - 1] if j else 0, ends[j])
            idx, ref, ref_norm = idx_all[sl], val_all[sl], float(norm_all[j])
            if ref_norm == 0.0:
                assert float(np.abs(g).max()) == 0.0, key
                continue
            err = float(np.linalg.norm(g[idx] - ref) / max(np.linalg.norm(ref), 1e-30))
            errs[key] = err
            # 3e-3 (the gate of tests/test_gpu_backward.py) plus what fp32 arithmetic itself leaves uncertain for this loss:
            # cond = how far the reference's own fp32 gradient is from the same reference run in float64, on these entries
            # (~1e-5 for most tensors; up to 2 % for mean(disp) over nearly empty rays, whose gradient grows like 1 / acc).
            # Two fp32 evaluations may each be that far from the exact value.
            cond = float(cond_all[j])
            assert err < 3e-3 + 2 * cond, (key, err, cond)
            assert abs(np.linalg.norm(g.astype(np.float64)) - ref_norm) <= (5e-3 + 2 * cond) * ref_norm, key
    _record(f"exact_vs_reference_{case}_{loss_name}", {"median": float(np.median(list(errs.values()))), "worst": max(errs.values())})
    assert np.median(list(errs.values())) < 3e-3


# ---- 4. tensor-core pass: dL/draw and the loss scale ----------------------------------------------------------------------

SEED_SETS = [("rgb_map",), ("acc_map",), ("rgb_map", "acc_map", "raw"), ("disp_map",), ("rgb_map", "disp_map", "acc_map", "depth_map", "weights", "raw")]


@pytest.mark.parametrize("keys", SEED_SETS, ids=["+".join(k) for k in SEED_SETS])
def test_tensor_core_pass_draw_and_loss_scale(G, keys):
    """one training-mode pass (view directions, 256 rays x 96 samples), then nerf_b200_march_bwd_tc_outs: the pass's dL/draw and
    amax in its workspace against the restatement; with rgb_map alone both equal what nerf_b200_march_bwd_tc leaves, bit for bit."""
    from nerf_pytorch_b200 import api
    lib = G._lib.load()
    N, S = 256, 96
    sb = G.synth.ray_batch("lego", N, seed=8)
    packed = G.O.pack_rays(400, 400, sb["K"], sb["rays"][0], sb["rays"][1], False, 2.0, 6.0, True).astype(np.float32)
    t = np.linspace(0., 1., S, dtype=np.float32)
    z = (packed[:, 6:7] * (1 - t) + packed[:, 7:8] * t).astype(np.float32)
    net = G.make_net(_trained()[1])             # acc spans 0..1 (a random net's rays are opaque: acc = 1, an ~0 acc gradient)
    n, pk = net.net_params(), net.packed()
    cfg = G._lib.NerfRenderCfg()
    cfg.N_samples, cfg.multires, cfg.multires_views, cfg.white_bkgd, cfg.ray_stride = S, 10, 4, 1, 11
    rays, zz = G.dev(packed), G.dev(z)
    raw = torch.zeros((N, S, 4), device=G.DEV)
    out = G._lib.NerfPassOut(None, None, None, None, None, G.ptr(raw))
    ws_f = torch.empty(lib.nerf_b200_march_workspace_bytes(N, S), dtype=torch.uint8, device=G.DEV)
    sv, act, mask = api._train_save(lib, N, S, n, G.DEV)
    G._lib.check(lib.nerf_b200_march_train(G.ptr(rays), G.ptr(zz), None, N, S, C.byref(n), G.ptr(pk), C.byref(cfg), C.byref(out),
                                           G.ptr(ws_f), ws_f.numel(), C.byref(sv), G.stream()), "march_train")
    rng = np.random.default_rng(4)
    seeds = {"rgb_map": rng.standard_normal((N, 3)) * 1e-3, "disp_map": rng.standard_normal(N) * 1e-2, "acc_map": rng.standard_normal(N) * 1e-2,
             "depth_map": rng.standard_normal(N) * 1e-3, "weights": rng.standard_normal((N, S)) * 1e-4, "raw": rng.standard_normal((N, S, 4)) * 1e-4}
    seeds = {k: G.dev(seeds[k].astype(np.float32)) for k in keys}
    lay = (C.c_int64 * 12)()
    G._lib.check(lib.nerf_b200_march_bwd_tc_layout(N, S, C.byref(n), lay), "layout")
    ws_bytes = lib.nerf_b200_march_bwd_tc_workspace_bytes(N, S, C.byref(n))

    def run(entry):
        ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=G.DEV)
        gbuf = api._grad_buffers(net)
        gs = net.grad_struct(gbuf)
        if entry == "old":
            G._lib.check(lib.nerf_b200_march_bwd_tc(G.ptr(rays), G.ptr(zz), None, N, S, C.byref(n), G.ptr(pk), C.byref(cfg), G.ptr(raw),
                                                    C.byref(sv), G.ptr(seeds["rgb_map"]), C.byref(gs), G.ptr(ws), ws_bytes, G.stream()), "old")
        else:
            og = G._lib.NerfOutGrads(**{k: G.ptr(v) for k, v in seeds.items()})
            G._lib.check(lib.nerf_b200_march_bwd_tc_outs(G.ptr(rays), G.ptr(zz), None, N, S, C.byref(n), G.ptr(pk), C.byref(cfg), G.ptr(raw),
                                                         C.byref(sv), C.byref(og), C.byref(gs), G.ptr(ws), ws_bytes, G.stream()), "outs")
        torch.cuda.synchronize()
        base = (-ws.data_ptr()) % 1024
        d_raw = ws[base + lay[0]: base + lay[0] + N * S * 16].view(torch.float32).reshape(N, S, 4).clone()
        amax = ws[base + lay[9]: base + lay[9] + 4].view(torch.float32).item()
        return d_raw, amax, gbuf

    d_raw, amax, _ = run("outs")
    ref = OG.adjoint(raw.cpu(), torch.from_numpy(z), torch.from_numpy(packed[:, 3:6]), True, {k: v.cpu() for k, v in seeds.items()})
    err = rel_l2(d_raw.cpu().numpy(), ref.numpy())
    ref_amax = OG.loss_scale_amax(raw.cpu(), torch.from_numpy(z), torch.from_numpy(packed[:, 3:6]), True, {k: v.cpu() for k, v in seeds.items()})
    _record("tc_stage_" + "+".join(keys), {"d_raw": err, "amax": amax, "amax_ref": ref_amax})
    assert err < 1e-4, err
    if "disp_map" in keys or "depth_map" in keys:      # products of the ray's fp32 depth / acc: the scale itself is exact
        assert abs(amax - ref_amax) <= 1e-4 * ref_amax and tc_emul.loss_scale(amax) == tc_emul.loss_scale(ref_amax), (amax, ref_amax)
    else:                                              # a max of the seeds themselves: exact
        assert amax == np.float32(ref_amax), (amax, ref_amax)
    if keys == ("rgb_map",):
        d_old, amax_old, g_old = run("old")
        d_new, amax_new, g_new = run("outs")
        assert torch.equal(d_old, d_new) and amax_old == amax_new
        assert amax_old == float(seeds["rgb_map"].abs().max())


# ---- 5. tensor-core vs exact backward on the same fp16 forward ------------------------------------------------------------

def _budget(devs):
    """the fp16 budget of the end-to-end tests (tests/test_gpu_train.py)"""
    med, worst = float(np.median(list(devs.values()))), max(devs.values())
    return med < 3e-2 and worst < 1.5e-1, med, worst


def _vs_exact(g_tc, g_ex):
    devs = {}
    for key, ge in g_ex.items():
        gt = g_tc[key]
        if not bool(torch.isfinite(ge).all()):        # NaN in the reference's arithmetic too (disp of an acc = 0 ray)
            assert torch.equal(torch.isnan(gt), torch.isnan(ge)), key
            continue
        assert torch.isfinite(gt).all(), key
        if float(ge.norm()) == 0.0:
            assert float(gt.abs().max()) == 0.0, key
            continue
        devs[f"{key[0]}.{key[1]}"] = float((gt - ge).norm() / ge.norm())
    return devs


NAMES = ["nerf_b200_render_rays_bwd_tc", "nerf_b200_render_rays_bwd_tc_outs", "nerf_b200_march_bwd_tc", "nerf_b200_march_bwd_tc_outs",
         "nerf_b200_march_bwd", "nerf_b200_march_bwd_outs"]


@pytest.mark.parametrize("loss_name", OG.LOSSES)
@pytest.mark.parametrize("case", CASES)
def test_tensor_core_matches_exact_same_forward(G, FX, monkeypatch, case, loss_name):
    lib = G._lib.load()
    with monkeypatch.context() as mp:
        spy = _Spy(mp, lib, NAMES)
        l_tc, n_tc = _render_case(G, FX, case, loss_name, "tc_fp16", "tc")
    # L_raw reads only the fine pass's raw: the coarse pass has no seed and does not run
    entry = "nerf_b200_march_bwd_tc_outs" if loss_name == "raw" else "nerf_b200_render_rays_bwd_tc_outs"
    assert spy.calls[entry] == 1 and sum(spy.calls.values()) == 1, spy.calls
    l_ex, n_ex = _render_case(G, FX, case, loss_name, "tc_fp16", "exact")
    assert l_tc == l_ex or (np.isnan(l_tc) and np.isnan(l_ex))
    devs = _vs_exact(_grads(n_tc), _grads(n_ex))
    ok, med, worst = _budget(devs)
    _record(f"tc_vs_exact_{case}_{loss_name}", {"median": med, "worst": worst})
    assert ok, (med, worst, devs)


@pytest.mark.parametrize("option", ["acc_only_fine", "coarse_only", "shared_net", "rgb_only"])
def test_tensor_core_render_options(G, FX, monkeypatch, option):
    """a loss without rgb (g_rgb absent), N_importance = 0, network_fine=None; and an rgb-only loss, which keeps the rgb entry point"""
    lib = G._lib.load()
    case = "a"
    runs = {}
    for bwd in ("tc", "exact"):
        nets = _nets(G, case)
        over = {}
        if option == "coarse_only":
            over = dict(N_importance=0)
        if option == "shared_net":
            nets[1] = None
        G.nb.set_backward(bwd)
        try:
            with monkeypatch.context() as mp:
                spy = _Spy(mp, lib, NAMES)
                o = _opts(case)
                o.update(over)
                rgb, disp, acc, ex = G.nb.render(int(FX["a_H"]), int(FX["a_W"]), FX["a_K"], rays=G.dev(FX["a_rays"]), ndc=False, near=2., far=6.,
                                                 network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64,
                                                 white_bkgd=True, retraw=True, **o)
                t_acc, target = G.dev(FX["a_t_acc"]), G.dev(FX["a_target"])
                if option == "acc_only_fine":
                    loss = torch.mean((acc - t_acc) ** 2)
                elif option == "rgb_only":
                    loss = torch.mean((rgb - target) ** 2) + torch.mean((ex["rgb0"] - target) ** 2)
                else:
                    ex0 = ex if "acc0" in ex else dict(ex, rgb0=rgb, disp0=disp, acc0=acc)
                    loss = OG.loss_of("all", rgb, disp, acc, ex0, target, t_acc)
                loss.backward()
        finally:
            G.nb.set_backward("tc")
        torch.cuda.synchronize()
        runs[bwd] = (spy.calls, _grads(nets))
    calls = runs["tc"][0]
    if option == "rgb_only":
        assert calls["nerf_b200_render_rays_bwd_tc"] == 1 and sum(calls.values()) == 1, calls
    elif option in ("acc_only_fine", "coarse_only"):
        assert calls["nerf_b200_march_bwd_tc_outs"] == 1 and sum(calls.values()) == 1, calls
    else:
        assert calls["nerf_b200_render_rays_bwd_tc_outs"] == 1 and sum(calls.values()) == 1, calls
    ex_calls = runs["exact"][0]
    assert ex_calls["nerf_b200_march_bwd" if option == "rgb_only" else "nerf_b200_march_bwd_outs"] >= 1, ex_calls
    devs = _vs_exact(runs["tc"][1], runs["exact"][1])
    ok, med, worst = _budget(devs)
    _record(f"tc_vs_exact_option_{option}", {"median": med, "worst": worst})
    assert ok, (med, worst, devs)


# ---- 6. 4096 rays ---------------------------------------------------------------------------------------------------------

def test_full_batch_l_all_repeatable_and_within_budget(G):
    sb = G.synth.ray_batch("lego", 4096, seed=3)
    rng = np.random.default_rng(5)
    fx = {"x_H": 400, "x_W": 400, "x_K": sb["K"], "x_rays": sb["rays"], "x_ndc": False, "x_near": 2., "x_far": 6., "x_white_bkgd": True,
          "x_target": rng.random((4096, 3), dtype=np.float32), "x_t_acc": rng.random(4096, dtype=np.float32)}
    opts = dict(N_importance=128, perturb=0., raw_noise_std=0., pytest=False, use_viewdirs=True)
    mk = lambda: [G.make_net(G.synth.nerf_state(0)), G.make_net(G.synth.nerf_state(1))]
    runs = [_render_case(G, fx, "x", "all", "tc_fp16", "tc", nets=mk(), **opts) for _ in range(3)]
    gs = [_grads(n) for _, n in runs]
    rep = max(float((g[k] - gs[0][k]).norm() / gs[0][k].norm().clamp_min(1e-30)) for g in gs[1:] for k in gs[0])
    _, n_ex = _render_case(G, fx, "x", "all", "tc_fp16", "exact", nets=mk(), **opts)
    devs = _vs_exact(gs[0], _grads(n_ex))
    ok, med, worst = _budget(devs)
    _record("full_batch_4096_l_all", {"repeat_max": rep, "median": med, "worst": worst})
    assert rep < 1e-4, rep
    assert ok, (med, worst, devs)
