"""Training is reproducible to the bit: with the same inputs, weights and torch seeds, every parameter gradient of loss.backward()
(through render(), render_rays() and raw2outputs(), on both backward paths) and every FusedTrainStep state are identical on every
run, whatever else runs on the GPU and whatever the library's buffers held before."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


def bits(t):
    """the tensor's bit pattern (NaNs compare equal to themselves)"""
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_same_bits(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(bits(x), bits(y)), f"{what}: tensor {i} differs in {int((bits(x) != bits(y)).sum())} elements"


def _nets(G, views, shared):
    from oracle import noviews
    if views:
        nets = [G.make_net(G.synth.nerf_state(0)), G.make_net(G.synth.nerf_state(1))]
    else:
        nets = [G.make_net(noviews.nerf_state_noviews(k), use_viewdirs=False) for k in (0, 1)]
    return [nets[0], None] if shared else nets


def _loss(rgb, disp, acc, ex, target, outputs):
    terms = [rgb] + ([ex["rgb0"]] if "rgb0" in ex else [])
    loss = sum(torch.mean((x - target) ** 2) for x in terms)
    if outputs == "all":
        for d, a in ((disp, acc),) + (((ex["disp0"], ex["acc0"]),) if "disp0" in ex else ()):
            loss = loss + 0.1 * torch.mean(torch.where(torch.isfinite(d), d, torch.zeros_like(d))) + torch.mean((a - 0.5) ** 2)
        raw = ex["raw"]
        loss = loss + 1e-3 * (torch.mean(torch.relu(raw[..., 3])) + torch.mean(raw[..., :3] ** 2))
    return loss


# (name, scene, N, N_samples, N_importance, perturb, raw_noise_std)
CASES = [
    ("config2", "lego", 4096, 64, 128, 1., 0.),          # the benchmark's shape
    ("n1024", "lego", 1024, 64, 128, 1., 0.),            # every shipped config's batch
    ("fern_noise", "fern", 1024, 64, 64, 1., 1.),
    ("n37_s70", "lego", 37, 70, 0, 0., 0.),              # S not a multiple of 64, a partial last CTA
    ("s1", "lego", 700, 1, 0, 0., 0.),                   # many rays per tile
    ("s300", "lego", 150, 300, 0, 1., 0.),               # rays straddling tiles and super-tiles
    ("s1024", "lego", 40, 1024, 0, 0., 0.),              # rays over four super-tiles
]


def _render_grads(G, case, nets, outputs, mode, views, seed=0):
    _, scene, N, Sc, Ni, perturb, noise = case
    sb = G.synth.ray_batch(scene, N, seed=11)
    params = [p for n in nets if n is not None for p in n.parameters()]
    for p in params:
        p.grad = None
    G.nb.set_backward(mode)
    try:
        torch.manual_seed(seed)
        target = torch.rand((N, 3), device=G.DEV)
        rgb, disp, acc, ex = G.nb.render(sb["H"], sb["W"], sb["K"], chunk=32768, rays=G.dev(sb["rays"]), ndc=sb["ndc"], near=sb["near"],
                                         far=sb["far"], use_viewdirs=views, network_fn=nets[0], network_fine=nets[1],
                                         network_query_fn=G.query_fn(), N_samples=Sc, N_importance=Ni, perturb=perturb,
                                         white_bkgd=sb["white_bkgd"], raw_noise_std=noise, retraw=True)
        loss = _loss(rgb, disp, acc, ex, target, outputs)
        loss.backward()
    finally:
        G.nb.set_backward("tc")
    torch.cuda.synchronize()
    grads = [p.grad.detach().clone() for p in params]
    assert torch.isfinite(loss)
    if outputs == "rgb":      # (disp_map's gradient is NaN on a ray with acc = 0, as in the reference: compared by bits below)
        assert all(torch.isfinite(g).all() for g in grads)
    return [loss.detach().clone()] + grads


def _busy(n=30):
    """an ordinary workload on another stream of this process, still running when the caller's work starts"""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = torch.randn(4096, 4096, device="cuda")
        for _ in range(n):
            a = torch.tanh(a @ a * (1.0 / 64))
    return s, a


VARIANTS = [(views, shared, outputs) for views in (True, False) for shared in (False, True) for outputs in ("rgb", "all")]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_render_backward_repeats_bitwise(G, case):
    """Each case twice from the same weights and seed; the second run while a matmul loop occupies the GPU from another stream.
    Networks with and without view directions, a separate or shared (network_fine=None) fine net, rgb-only and all-output losses,
    the tensor-core backward and (at small N x S) the exact one."""
    small = case[2] * (case[3] + case[4]) <= 50000
    for views, shared, outputs in VARIANTS:
        if shared and case[4] == 0:
            continue                                                  # coarse-only: no fine net to share
        for mode in ("tc", "exact") if small else ("tc",):
            nets = _nets(G, views, shared or case[4] == 0)
            first = _render_grads(G, case, nets, outputs, mode, views)
            s, _ = _busy()
            second = _render_grads(G, case, nets, outputs, mode, views)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            assert_same_bits(first, second, f"{case[0]} views={views} shared={shared} {outputs} {mode}")


def test_render_rays_and_raw2outputs_repeat_bitwise(G):
    sb = G.synth.ray_batch("lego", 512, seed=5)
    packed = torch.from_numpy(G.O.pack_rays(400, 400, sb["K"], sb["rays"][0], sb["rays"][1], False, 2., 6., True).astype(np.float32)).to(G.DEV)
    nets = _nets(G, True, False)

    def run_rays():
        for n in nets:
            n.zero_grad(set_to_none=True)
        torch.manual_seed(3)
        ret = G.nb.render_rays(packed, nets[0], G.query_fn(), 64, retraw=True, perturb=1., N_importance=64, network_fine=nets[1],
                               white_bkgd=True, raw_noise_std=1.)
        loss = ret["rgb_map"].square().mean() + ret["rgb0"].square().mean() + ret["acc_map"].mean() + 1e-3 * ret["raw"].square().mean()
        loss.backward()
        return [loss.detach()] + [p.grad.clone() for n in nets for p in n.parameters()]

    assert_same_bits(run_rays(), run_rays(), "render_rays")

    def run_r2o():
        torch.manual_seed(4)
        raw = torch.randn(2000, 96, 4, device=G.DEV).requires_grad_(True)
        z = torch.sort(torch.rand(2000, 96, device=G.DEV) * 4 + 2, -1)[0]
        d = torch.randn(2000, 3, device=G.DEV)
        rgb, disp, acc, w, depth = G.nb.raw2outputs(raw, z, d, raw_noise_std=1., white_bkgd=True)
        (rgb.square().mean() + acc.mean() + w.square().mean() + depth.mean()).backward()
        return [raw.grad.clone()]

    assert_same_bits(run_r2o(), run_r2o(), "raw2outputs")


# ---- the C ABI with poisoned buffers ---------------------------------------------------------------------------------

def _tc_pass(G, net, rays, z, g_rgb, fill):
    """training-mode forward + tensor-core backward of one pass with workspace and records pre-filled with `fill` -> grads, ws"""
    from nerf_pytorch_b200 import _lib, api
    lib = _lib.load()
    N, S = z.shape
    n = net.net_params()
    c = G.cfg(S, rays.shape[1])
    o = {k: torch.zeros(s, device=G.DEV) for k, s in (("rgb", (N, 3)), ("disp", (N,)), ("acc", (N,)), ("w", (N, S)), ("raw", (N, S, 4)))}
    out = _lib.NerfPassOut(G.ptr(o["rgb"]), G.ptr(o["disp"]), G.ptr(o["acc"]), C.c_void_p(0), G.ptr(o["w"]), G.ptr(o["raw"]))
    fws = lib.nerf_b200_march_workspace_bytes(N, S)
    fw = torch.full((fws,), fill, dtype=torch.uint8, device=G.DEV)
    sv, act, mask = api._train_save(lib, N, S, n, G.DEV)
    act.fill_(fill); mask.fill_(fill)
    _lib.check(lib.nerf_b200_march_train(G.ptr(rays), G.ptr(z), None, N, S, C.byref(n), G.ptr(net.packed()), C.byref(c), C.byref(out),
                                         G.ptr(fw), fws, C.byref(sv), G.stream()), "march_train")
    grads = {k: torch.zeros_like(p) for k, p in net.named_parameters()}
    gs = net.grad_struct(grads)
    bws = lib.nerf_b200_march_bwd_tc_workspace_bytes(N, S, C.byref(n))
    ws = torch.full((bws + 1024,), fill, dtype=torch.uint8, device=G.DEV)
    _lib.check(lib.nerf_b200_march_bwd_tc(G.ptr(rays), G.ptr(z), None, N, S, C.byref(n), G.ptr(net.packed()), C.byref(c), G.ptr(o["raw"]),
                                          C.byref(sv), G.ptr(g_rgb), C.byref(gs), G.ptr(ws), bws + 1024, G.stream()), "march_bwd_tc")
    torch.cuda.synchronize()
    base = (ws.data_ptr() + 1023) // 1024 * 1024 - ws.data_ptr()
    return [grads[k] for k in sorted(grads)], ws.cpu().numpy()[base:]


def _pass_inputs(G, N, S, views=True):
    sb = G.synth.ray_batch("lego", N, seed=2)
    rays = torch.from_numpy(G.O.pack_rays(400, 400, sb["K"], sb["rays"][0], sb["rays"][1], False, 2., 6., views).astype(np.float32)).to(G.DEV)
    t = torch.linspace(0., 1., S, device=G.DEV)
    z = (rays[:, 6:7] * (1 - t) + rays[:, 7:8] * t).contiguous()
    g = torch.randn((N, 3), device=G.DEV, generator=torch.Generator(G.DEV).manual_seed(S))
    return rays, z, g


BUFFER_CASES = [(4096, 192, True), (37, 70, True), (700, 1, True), (150, 300, True), (40, 1024, True), (4096, 192, False)]


@pytest.mark.parametrize("N,S,views", BUFFER_CASES, ids=[f"{n}-{s}" + ("" if v else "-noviews") for n, s, v in BUFFER_CASES])
def test_buffer_contents_do_not_matter_and_dsum_is_exact(G, N, S, views):
    """0x00- and 0xFF-filled workspace and records give the same gradient bits, with view directions (d_hv seed) and without
    (dA_seed_output_kernel).  The per-ray sums of d_hv (dsum) equal float64 sums of the decoded d_hv images to within fp32
    summation error."""
    import tc_records as R
    from nerf_pytorch_b200 import _lib
    from oracle import noviews
    net = G.make_net(G.synth.nerf_state(0)) if views else G.make_net(noviews.nerf_state_noviews(0, True), use_viewdirs=False)
    rays, z, g = _pass_inputs(G, N, S, views)
    ga, ws = _tc_pass(G, net, rays, z, g, 0x00)
    gb, _ = _tc_pass(G, net, rays, z, g, 0xFF)
    assert all(torch.isfinite(x).all() for x in ga)
    assert_same_bits(ga, gb, f"N={N} S={S} views={views} poisoned buffers")
    if not views:
        return
    plan = R.Plan(_lib.load(), N, S, net.net_params())
    amax = float(ws[plan.off_amax:plan.off_amax + 4].view(np.float32)[0])
    scale = 2.0 ** np.floor(np.log2(np.float32(2048.0) / np.float32(amax)))
    dhv = R.gather_image(ws[plan.off_grad:], plan, plan.rec_grad, 0, 128).astype(np.float64)
    per_ray = dhv.reshape(N, S, 128)
    ref = per_ray.sum(1) / scale
    bound = (S + 1) * 2.0 ** -24 * np.abs(per_ray).sum(1) / scale + 1e-30
    dsum = ws[plan.off_dsum:plan.off_dsum + N * 128 * 4].view(np.float32).reshape(N, 128).astype(np.float64)
    assert np.all(np.abs(dsum - ref) <= bound), float(np.max(np.abs(dsum - ref) - bound))


def test_deterministic_algorithms_mode_same_bits(G):
    """render() under torch.use_deterministic_algorithms(True) with uninitialised memory filled: no torch op on the host path
    raises, and the gradients are the bits of a normal run."""
    import torch.utils.deterministic as tud
    case = CASES[1]
    nets = _nets(G, True, False)
    normal = _render_grads(G, case, nets, "all", "tc", True)
    fill = tud.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True)
    tud.fill_uninitialized_memory = True
    try:
        det = _render_grads(G, case, nets, "all", "tc", True)
    finally:
        torch.use_deterministic_algorithms(False)
        tud.fill_uninitialized_memory = fill
    assert_same_bits(normal, det, "deterministic-algorithms mode")


@pytest.mark.parametrize("views", [True, False])
@pytest.mark.parametrize("N", [1024, 4096])
def test_fused_train_step_bitwise(G, N, views):
    """Two FusedTrainStep instances from the same weights and seed: after 20 graph-replayed steps with perturb and noise, the
    flat parameters, Adam moments and step state are identical."""
    from nerf_pytorch_b200.trainer import FusedTrainStep
    sb = G.synth.ray_batch("lego", N, seed=6)
    rays_h = torch.from_numpy(sb["rays"]).pin_memory()
    tgt_h = torch.from_numpy(np.random.default_rng(1).random((N, 3), dtype=np.float32)).pin_memory()
    runs = []
    for _ in range(2):
        nets = _nets(G, views, False)
        kw = dict(network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64, N_importance=128, perturb=1.,
                  white_bkgd=True, raw_noise_std=1., use_viewdirs=views, ndc=False, lindisp=False, near=2., far=6.)
        torch.manual_seed(9)
        tr = FusedTrainStep(400, 400, sb["K"], N, kw, use_graph=True)
        losses = torch.tensor([tr(rays_h, tgt_h) for _ in range(20)])
        torch.cuda.synchronize()
        runs.append([tr.flat_p.clone(), tr.m.clone(), tr.v.clone(), tr.state.clone(), losses])
    assert np.all(np.isfinite(runs[0][4].numpy()))
    assert_same_bits(runs[0], runs[1], f"FusedTrainStep N={N} views={views}")
