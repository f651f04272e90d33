"""The tensor-core training path for networks WITHOUT view directions (use_viewdirs=False: output_linear head, the reference's
default, run_nerf.py:467 / :187): training-mode forward records, the backward stage by stage against the quantisation-aware
restatement (oracle/noviews.py), end to end against the exact mode and the reference's autograd
(tests/golden/lego_noviews_grads.npz), the render() options, FusedTrainStep and the C ABI.  Measured deviations are appended
to parity_train_noviews.json in $NERF_B200_PARITY_DIR (default: a nerf_b200_parity directory under the system's temporary
directory)."""
import ctypes as C
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2

pytestmark = pytest.mark.gpu

D = 8


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


def _record(name, value):
    out_dir = os.environ.get("NERF_B200_PARITY_DIR") or os.path.join(tempfile.gettempdir(), "nerf_b200_parity")
    path = os.path.join(out_dir, "parity_train_noviews.json")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    data = {}
    if os.path.isfile(path):
        with open(path) as f:
            data = json.load(f)
    data[name] = value
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def _net(G, seed, sharpen=False, output_ch=5):
    from oracle import noviews
    state = noviews.nerf_state_noviews(seed, sharpen, output_ch=output_ch)
    return G.make_net(state, use_viewdirs=False, output_ch=output_ch), state


def _inputs(G, N, S, seed, sharpen=False):
    sb = G.synth.ray_batch("lego", N, seed=seed)
    packed = G.O.pack_rays(400, 400, sb["K"], sb["rays"][0], sb["rays"][1], False, 2.0, 6.0, False).astype(np.float32)
    assert packed.shape == (N, 8)
    net, state = _net(G, seed % 2, sharpen)
    t = np.linspace(0., 1., S, dtype=np.float32)
    z = (packed[:, 6:7] * (1 - t) + packed[:, 7:8] * t).astype(np.float32)
    if S > 64:                                   # uneven spacing like a fine pass
        rng = np.random.default_rng(seed)
        z = np.sort(z + rng.uniform(-0.01, 0.01, z.shape).astype(np.float32), -1)
    return packed, z, state, net


def _emul_forward(state, packed, z):
    from oracle import noviews
    pts = (packed[:, None, 0:3] + packed[:, None, 3:6] * z[..., None]).reshape(-1, 3)
    sd = {k: torch.from_numpy(v) for k, v in state.items()}
    return noviews.forward_noviews(sd, torch.from_numpy(pts)), sd


@pytest.mark.parametrize("N,S", [(100, 64), (37, 192), (50, 40)])
def test_training_forward_records_noviews(G, N, S):
    """The training instantiation returns what inference returns, bit for bit, and its records decode to the fp16 encodings,
    every h_l (h_{D-1} included, which inference does not store) and the sign masks."""
    import tc_records as R
    packed, z, state, net = _inputs(G, N, S, seed=5)
    rays8, zd = G.dev(packed), G.dev(z)
    o_inf, _, _ = G.march(net, rays8, zd, train=False)
    o_tr, act, mask = G.march(net, rays8, zd, train=True)
    for k in ("rgb", "disp", "acc", "w", "raw"):                       # bit patterns: disp is NaN where acc = 0 (run_nerf.py:299)
        assert torch.equal(o_inf[k].view(torch.int32), o_tr[k].view(torch.int32)), k
    plan = R.Plan(G._lib.load(), N, S, net.net_params())
    A, Mk = act.cpu().numpy(), mask.cpu().numpy()
    em, _ = _emul_forward(state, packed, z)
    stats = {}
    enc = R.gather_image(A, plan, plan.rec_act, 0, 64)
    ref_enc = np.concatenate([em["enc16"].numpy(), np.zeros((N * S, 1))], 1)
    assert not np.isnan(enc).any()
    stats["enc_close"] = float(np.mean(np.isclose(enc, ref_enc, rtol=2e-3, atol=1e-4)))
    assert stats["enc_close"] > 0.995, stats
    for l in range(D):
        h = R.gather_image(A, plan, plan.rec_act, 16384 + l * 65536, 256)
        assert not np.isnan(h).any(), l
        stats[f"h{l}_rel"] = rel_l2(h, em["h16"][l].numpy())
        assert stats[f"h{l}_rel"] < 2e-3, (l, stats)
        m = R.gather_mask(Mk, plan, l, D)
        stats[f"mask{l}_mismatch"] = float(np.mean(m != (h > 0)))
        assert stats[f"mask{l}_mismatch"] < 2e-4, (l, stats)              # fp16 underflow of a positive pre-activation only
    stats["raw_rel"] = rel_l2(o_tr["raw"].cpu().numpy().reshape(-1, 4), em["raw"].numpy())
    assert stats["raw_rel"] < 2e-3, stats
    _record(f"records_N{N}_S{S}", stats)


@pytest.mark.parametrize("N,S,sharpen", [(100, 64, False), (37, 192, False), (64, 64, True), (50, 40, False)])
def test_backward_stages_match_emulation_noviews(G, N, S, sharpen):
    """dL/draw, the dA_{D-1} seed (output_linear head), each dgrad step's fp16 tile image and every gradient tensor, output_linear's
    included -- given the CUDA forward's own records -- against the same arithmetic in torch (oracle/noviews.py)."""
    import tc_records as R
    from oracle import noviews
    from oracle import tc_emul as E
    packed, z, state, net = _inputs(G, N, S, seed=7, sharpen=sharpen)
    rays8, zd = G.dev(packed), G.dev(z)
    o, act, mask = G.march(net, rays8, zd, train=True)
    rng = np.random.default_rng(11)
    g_rgb = ((rng.random((N, 3), dtype=np.float32) - 0.5) * (4.0 / (3 * N))).astype(np.float32)
    grads, ws = G.march_bwd_tc(net, rays8, zd, o["raw"], act, mask, G.dev(g_rgb))
    plan = R.Plan(G._lib.load(), N, S, net.net_params())
    M = N * S
    A, Mk = act.cpu().numpy(), mask.cpu().numpy()
    stats = {}
    d_raw = ws[plan.off_draw:plan.off_draw + M * 16].view(np.float32).reshape(M, 4)
    amax = float(ws[plan.off_amax:plan.off_amax + 4].view(np.float32)[0])
    assert abs(amax - float(np.abs(g_rgb).max())) < 1e-12
    scale = E.loss_scale(amax)
    ref_draw = E.composite_adjoint(o["raw"].cpu(), torch.from_numpy(z), torch.from_numpy(packed[:, 3:6]), torch.from_numpy(g_rgb), True).numpy().reshape(M, 4)
    stats["d_raw_rel"] = rel_l2(d_raw, ref_draw)
    assert stats["d_raw_rel"] < 1e-4, stats
    acts = {"enc16": torch.from_numpy(R.gather_image(A, plan, plan.rec_act, 0, 64)).double(),
            "h16": [torch.from_numpy(R.gather_image(A, plan, plan.rec_act, 16384 + l * 65536, 256)).double() for l in range(D)]}
    masks = {"h": [torch.from_numpy(R.gather_mask(Mk, plan, l, D)).double() for l in range(D)]}
    sd = {k: torch.from_numpy(v) for k, v in state.items()}
    ref_g, st = noviews.backward_noviews(sd, acts, masks, torch.from_numpy(d_raw).double(), scale)
    Gr = ws[plan.off_grad:plan.off_grad + plan.n_tiles * plan.rec_grad]
    for j in range(1, D + 1):                    # step 1: the seed dA_{D-1}; step j: dA_{D-j}
        img = R.gather_image(Gr, plan, plan.rec_grad, 32768 + j * 65536, 256)
        assert not np.isnan(img).any(), j
        stats[f"step{j}_rel"] = rel_l2(img, st["step"][j].numpy())
        assert stats[f"step{j}_rel"] < 2e-3, (j, stats)
    assert set(ref_g) == set(grads)
    for name, ref in ref_g.items():
        if float(ref.abs().max()) == 0.0:        # views_linears.0: not on the loss's graph
            assert not grads[name].any(), name
            continue
        e = rel_l2(grads[name].reshape(-1), ref.numpy().reshape(-1))
        stats["g_" + name] = e
        assert e < 2e-3, (name, e, stats)
    assert grads["output_linear.weight"][4].tolist() == [0.0] * 256 and grads["output_linear.bias"][4] == 0.0
    _record(f"bwd_stages_N{N}_S{S}_sharp{int(sharpen)}", stats)


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


def _render_loss(G, nets, sb, target, prec, backward, N_importance=128, perturb=0., raw_noise_std=0., pytest_draws=False):
    G.nb.set_precision(prec)
    G.nb.set_backward(backward)
    for n in nets:
        if n is not None:
            n.zero_grad(set_to_none=True)
    try:
        rgb, disp, acc, ex = G.nb.render(int(sb["H"]), int(sb["W"]), sb["K"], chunk=32768, rays=G.dev(sb["rays"]), ndc=bool(sb["ndc"]),
                                         near=float(sb["near"]), far=float(sb["far"]), use_viewdirs=False, network_fn=nets[0],
                                         network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64, N_importance=N_importance,
                                         perturb=perturb, white_bkgd=bool(sb["white_bkgd"]), raw_noise_std=raw_noise_std, retraw=True,
                                         pytest=pytest_draws)
        t = G.dev(target)
        loss = G.nb.img2mse(rgb, t)
        if N_importance > 0:
            loss = loss + G.nb.img2mse(ex["rgb0"], t)
        loss.backward()
    finally:
        G.nb.set_precision("tc_fp16")
        G.nb.set_backward("tc")
    torch.cuda.synchronize()
    return float(loss.item())


def _grads(nets):
    return {(k, name): p.grad.detach().double().cpu() for k, n in enumerate(nets) if n is not None for name, p in n.named_parameters()}


def _vs_exact(g_tc, g_ex):
    """per-tensor rel-L2 of the tensor-core gradients against the exact ones; tensors off the loss's graph must be exactly zero"""
    devs = {}
    for key, ge in g_ex.items():
        gt = g_tc[key]
        assert torch.isfinite(gt).all(), key
        if float(ge.norm()) == 0.0:
            assert float(gt.abs().max()) == 0.0, key
            continue
        devs[f"{key[0]}.{key[1]}"] = float((gt - ge).norm() / ge.norm())
    return devs


def _budget(devs):
    """the fp16 budget of the view-direction path's end-to-end tests (tests/test_gpu_train.py)"""
    med, worst = float(np.median(list(devs.values()))), max(devs.values())
    return med < 3e-2 and worst < 1.5e-1, med, worst


def _vs_reference(fx, tag, net):
    """per-tensor rel-L2 of the net's gradients at the fixture's sampled entries; parameters the reference leaves without a
    gradient (views_linears.0, not on the loss's graph) must have an all-zero one"""
    out = {}
    for name, p in net.named_parameters():
        g = p.grad.detach().cpu().numpy().reshape(-1)
        if f"g_{tag}_{name}_idx" not in fx:
            assert not g.any(), (tag, name)
            continue
        idx, ref = fx[f"g_{tag}_{name}_idx"], fx[f"g_{tag}_{name}_val"]
        out[name] = float(np.linalg.norm(g[idx] - ref) / max(np.linalg.norm(ref), 1e-12))
    return out


def test_tensor_core_gradients_end_to_end_noviews(G, monkeypatch):
    """render() + img2mse x 2 + loss.backward() under the default settings runs the training-mode forward and the tensor-core
    backward (not the exact one).  Its gradients match the exact backward taken on the same (fp16) forward, and the reference's
    autograd: the coarse net within the fp16 budget of the view-direction path, the fine net no further from the reference than
    the exact backward on that same forward is.  (The fine pass samples where the coarse pass's weights put it: the fp16 coarse
    forward moves those samples by ~5e-5 relative, and on this 24-ray batch that alone moves the fine net's fp32 gradients by
    ~11 % median -- a property of the forward, which this change does not touch.)"""
    fx = load_golden("lego_noviews_grads")
    assert not bool(fx["use_viewdirs"]) and int(fx["output_ch"]) == 5
    lib = G._lib.load()
    names = ["nerf_b200_render_rays_fwd_train", "nerf_b200_render_rays_bwd_tc", "nerf_b200_march_bwd", "nerf_b200_march_bwd_tc"]
    sw = int(fx["seed_w"])
    runs = {}
    for key, prec, bwd in (("tc", "tc_fp16", "tc"), ("tc_fwd_exact_bwd", "tc_fp16", "exact"), ("exact", "fp32", "exact")):
        nets = [_net(G, sw)[0], _net(G, sw + 1)[0]]
        with monkeypatch.context() as mp:
            spy = _Spy(mp, lib, names)
            loss = _render_loss(G, nets, fx, fx["target"], prec, bwd)
        if bwd == "tc":
            assert spy.calls == {"nerf_b200_render_rays_fwd_train": 1, "nerf_b200_render_rays_bwd_tc": 1, "nerf_b200_march_bwd": 0,
                                 "nerf_b200_march_bwd_tc": 0}, spy.calls
        else:
            assert spy.calls["nerf_b200_march_bwd"] == 2 and spy.calls["nerf_b200_render_rays_bwd_tc"] == 0, spy.calls
        runs[key] = (loss, nets)
    ref_loss = float(fx["loss"])
    assert abs(runs["tc"][0] - ref_loss) / ref_loss < 5e-4
    assert abs(runs["exact"][0] - ref_loss) / ref_loss < 1e-5
    same_fwd = _vs_exact(_grads(runs["tc"][1]), _grads(runs["tc_fwd_exact_bwd"][1]))
    vs_exact = _vs_exact(_grads(runs["tc"][1]), _grads(runs["exact"][1]))
    ref = {(tag, key): _vs_reference(fx, tag, runs[key][1][k]) for tag, k in (("c", 0), ("f", 1)) for key in ("tc", "tc_fwd_exact_bwd")}
    _record("e2e_lego_noviews_grads", {"tc_vs_exact_bwd_same_forward": same_fwd, "tc_vs_exact": vs_exact,
                                       "vs_reference": {f"{t}.{k}": v for (t, k), v in ref.items()}})
    ok, med, worst = _budget(same_fwd)
    print("no-view tensor-core backward vs exact backward on the same forward: median", med, "worst", worst)
    assert ok, (med, worst, same_fwd)
    c = ref[("c", "tc")]
    med, worst = float(np.median(list(c.values()))), max(c.values())
    print("coarse net vs reference autograd: median", med, "worst", worst)
    assert med < 3e-2 and worst < 1.5e-1, (med, worst, c)
    for name, e in ref[("f", "tc")].items():
        assert e < ref[("f", "tc_fwd_exact_bwd")][name] + 1e-2, (name, e, ref[("f", "tc_fwd_exact_bwd")][name])


def test_full_batch_tensor_core_gradients_noviews(G):
    """4096 rays x 64 + 128 (every CTA walks many super-tiles): three tensor-core evaluations agree with each other (atomics
    reorder sums: 1e-4) and with the exact backward within the fp16 budget."""
    sb = G.synth.ray_batch("lego", 4096, seed=3)
    target = np.random.default_rng(5).random((4096, 3), dtype=np.float32)
    runs = []
    for _ in range(3):
        nets = [_net(G, 0)[0], _net(G, 1)[0]]
        runs.append((_render_loss(G, nets, sb, target, "tc_fp16", "tc"), _grads(nets)))
    nets_ex = [_net(G, 0)[0], _net(G, 1)[0]]
    loss_ex = _render_loss(G, nets_ex, sb, target, "fp32", "exact")
    rep = []
    for key, g0 in runs[0][1].items():
        for _, other in runs[1:]:
            rep.append(float((other[key] - g0).norm() / g0.norm().clamp_min(1e-30)))
    devs = _vs_exact(runs[0][1], _grads(nets_ex))
    ok, med, worst = _budget(devs)
    _record("full_batch_4096", {"repeat_max": max(rep), "vs_exact_median": med, "vs_exact_max": worst,
                                "loss_rel": abs(runs[0][0] - loss_ex) / loss_ex})
    assert max(rep) < 1e-4, max(rep)
    assert abs(runs[0][0] - loss_ex) / loss_ex < 5e-4
    assert ok, (med, worst, devs)


@pytest.mark.parametrize("case", ["coarse_only", "shared_net", "perturb_noise", "fern_ndc"])
def test_render_options_noviews(G, case):
    """render() options, tensor-core backward vs exact backward: N_importance = 0 (output_ch = 4, coarse pass only),
    network_fine=None (both passes accumulate into one net), perturb = 1 with raw_noise_std = 1 (the pytest=True draws), and a
    fern-shaped NDC batch without white_bkgd."""
    kw = {}
    out_ch = 5
    if case == "coarse_only":
        kw["N_importance"], out_ch = 0, 4
    elif case == "perturb_noise":
        kw.update(perturb=1., raw_noise_std=1., pytest_draws=True)
    sb = G.synth.ray_batch("fern" if case == "fern_ndc" else "lego", 256, seed=12)
    target = np.random.default_rng(6).random((256, 3), dtype=np.float32)
    res = {}
    for prec, bwd in (("tc_fp16", "tc"), ("fp32", "exact")):
        nets = [_net(G, 2, output_ch=out_ch)[0], None if case in ("shared_net", "coarse_only") else _net(G, 3, output_ch=out_ch)[0]]
        loss = _render_loss(G, nets, sb, target, prec, bwd, **kw)
        res[bwd] = (loss, _grads(nets))
    devs = _vs_exact(res["tc"][1], res["exact"][1])
    ok, med, worst = _budget(devs)
    loss_rel = abs(res["tc"][0] - res["exact"][0]) / res["exact"][0]
    _record(f"options_{case}", {"loss_rel": loss_rel, "vs_exact_median": med, "vs_exact_max": worst})
    assert loss_rel < 5e-4, loss_rel
    assert ok, (case, med, worst, devs)


def _kwargs(G, nets):
    return dict(network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64, N_importance=128, perturb=0.,
                white_bkgd=True, raw_noise_std=0., use_viewdirs=False, ndc=False, lindisp=False, near=2., far=6.)


@pytest.mark.parametrize("use_graph", [True, False])
def test_fused_step_matches_autograd_adam_noviews(G, use_graph):
    """FusedTrainStep trains a no-view net ([N, 8] ray batch) and takes the steps of render() + autograd + torch.optim.Adam with the
    reference's host-side decay (run_nerf.py:760-784)."""
    from nerf_pytorch_b200.trainer import FusedTrainStep
    N, steps, lrate, decay = 200, 4, 5e-4, 0.002
    sb = G.synth.ray_batch("lego", N, seed=8)
    rays = G.dev(sb["rays"])
    target = G.dev(np.random.default_rng(2).random((N, 3), dtype=np.float32))
    nets_a = [_net(G, 0)[0], _net(G, 1)[0]]
    params = list(nets_a[0].parameters()) + list(nets_a[1].parameters())
    opt = torch.optim.Adam(params, lr=lrate, betas=(0.9, 0.999))
    kw = _kwargs(G, nets_a)
    losses_a, global_step = [], 0
    for _ in range(steps):
        rgb, _, _, ex = G.nb.render(400, 400, sb["K"], chunk=32768, rays=rays, retraw=True, **kw)
        opt.zero_grad()
        loss = G.nb.img2mse(rgb, target) + G.nb.img2mse(ex["rgb0"], target)
        loss.backward()
        opt.step()
        for pg in opt.param_groups:
            pg["lr"] = lrate * (0.1 ** (global_step / (decay * 1000)))          # run_nerf.py:779-783
        global_step += 1
        losses_a.append(float(loss))
    nets_b = [_net(G, 0)[0], _net(G, 1)[0]]
    init = [p.detach().clone() for n in nets_b for p in n.parameters()]
    tr = FusedTrainStep(400, 400, sb["K"], N, _kwargs(G, nets_b), lrate=lrate, lrate_decay=decay, use_graph=use_graph)
    assert tr.packed_rays.shape == (N, 8)
    for p, p0 in zip([p for n in nets_b for p in n.parameters()], init):
        assert torch.equal(p.detach(), p0)
    rays_h, tgt_h = rays.cpu().pin_memory(), target.cpu().pin_memory()
    losses_b = [tr(rays_h, tgt_h) for _ in range(steps)]
    assert tr.global_step == steps
    assert np.allclose(losses_a, losses_b, rtol=2e-4), (losses_a, losses_b)
    worst = 0.0
    for pa, pb, p0 in zip([p for n in nets_a for p in n.parameters()], [p for n in nets_b for p in n.parameters()], init):
        da, db = (pa.detach() - p0).cpu().numpy(), (pb.detach() - p0).cpu().numpy()
        if not da.any():                         # views_linears.0: never updated on either side
            assert not db.any()
            continue
        worst = max(worst, rel_l2(db, da))
    _record(f"fused_step_graph{int(use_graph)}", {"losses_autograd": losses_a, "losses_fused": losses_b, "update_worst": worst})
    assert worst < 5e-2, worst
    with torch.no_grad():
        a = G.nb.render(400, 400, sb["K"], rays=rays, **_kwargs(G, nets_a))[0]
        b = G.nb.render(400, 400, sb["K"], rays=rays, **_kwargs(G, nets_b))[0]
    assert rel_l2(b.cpu().numpy(), a.cpu().numpy()) < 2e-3


def test_c_abi_noviews_queries_and_mismatch(G):
    """The workspace / layout queries serve no-view nets; a coarse / fine use_viewdirs mismatch is refused by argument
    validation (error code and message, nothing launched)."""
    lib = G._lib.load()
    net_nv, _ = _net(G, 0)
    net_vd = G.make_net(G.synth.nerf_state(1))
    n_nv, n_vd = net_nv.net_params(), net_vd.net_params()
    N, Sc, Sf = 64, 64, 192
    assert lib.nerf_b200_march_bwd_tc_workspace_bytes(N, Sc, C.byref(n_nv)) > 0
    assert lib.nerf_b200_render_rays_bwd_tc_workspace_bytes(N, Sc, C.byref(n_nv), Sf, C.byref(n_nv)) > 0
    assert lib.nerf_b200_render_rays_bwd_tc_workspace_bytes(N, Sc, C.byref(n_nv), Sf, C.byref(n_vd)) == 0
    out = (C.c_int64 * 12)()
    assert lib.nerf_b200_march_bwd_tc_layout(N, Sc, C.byref(n_nv), out) == 0 and all(int(v) > 0 for v in out[2:9])
    # packed weights: the backward stream of a no-view net is the 8 (D - 1) pts-layer chunks (16 KB each)
    assert lib.nerf_b200_packed_bytes(C.byref(n_nv)) >= 8 * (D - 1) * 16384
    dummy = torch.zeros(1 << 16, device=G.DEV)
    cfg = G.cfg(Sc, 8)
    grads = [{k: torch.zeros_like(p) for k, p in n.named_parameters()} for n in (net_nv, net_vd)]
    gs = [net_nv.grad_struct(grads[0]), net_vd.grad_struct(grads[1])]
    sv = G._lib.NerfTrainSave(G.ptr(dummy), dummy.numel() * 4, G.ptr(dummy), dummy.numel() * 4)
    bp = [G._lib.NerfBwdPass(G.ptr(dummy), None, S, C.pointer(n), G.ptr(net.packed()), G.ptr(dummy), C.pointer(sv), G.ptr(dummy), C.pointer(g))
          for S, n, net, g in ((Sc, n_nv, net_nv, gs[0]), (Sf, n_vd, net_vd, gs[1]))]
    before = G.nb.launch_count()
    rc = lib.nerf_b200_render_rays_bwd_tc(G.ptr(dummy), N, C.byref(cfg), C.byref(bp[0]), C.byref(bp[1]), G.ptr(dummy), dummy.numel() * 4, G.stream())
    assert rc != 0
    assert b"use_viewdirs" in lib.nerf_b200_last_error()
    assert G.nb.launch_count() == before
    torch.cuda.synchronize()
