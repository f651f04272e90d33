"""FusedTrainStep and GraphedRender on any ray count up to the one they were built for.  A step of n < n_rays rays runs on the
first n rows of the step's buffers under a graph captured on first use, and takes exactly the step a FusedTrainStep built for n
rays takes: the same parameters, Adam moments, state and loss, bit for bit, with perturb and sigma noise on.  So the reference's
loop over shuffled rays, whose last batch of an epoch is short (run_nerf.py:717-726), runs on the fused step: graph and eager
steps agree bit for bit, the drop-in autograd loop agrees within test_gpu_trainer.py's gates, and a run interrupted before or
after a short batch resumes to the bits of the uninterrupted one."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu
LRATE, DECAY = 5e-4, 0.002                      # decay_steps = 2: a step count off by one changes the rate visibly
CAP, SHORT = 1024, 816                          # fern at factor 8 / llffhold 8 with N_rand 1024: the last batch has 816 rays


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_same_bits(a, b, what):
    assert len(a) == len(b)
    for name, x, y in zip(("flat_p", "m", "v", "state", "losses"), a, b):
        assert torch.equal(bits(x), bits(y)), f"{what}: {name} differs in {int((bits(x) != bits(y)).sum())} of {x.numel()} elements"


def _nets(G, views):
    from oracle import noviews
    if views:
        return [G.make_net(G.synth.nerf_state(k)) for k in (0, 1)]
    return [G.make_net(noviews.nerf_state_noviews(k), use_viewdirs=False) for k in (0, 1)]


def _kwargs(G, nets, views):
    return dict(network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64, N_importance=64, perturb=1.,
                white_bkgd=True, raw_noise_std=1., use_viewdirs=views, ndc=False, lindisp=False, near=2., far=6.)


def _step(G, views, n_rays, use_graph=True, nets=None):
    from nerf_pytorch_b200.trainer import FusedTrainStep
    H, W, K, _ = G.synth.lego_camera(400)
    nets = _nets(G, views) if nets is None else nets
    return FusedTrainStep(H, W, K, n_rays, _kwargs(G, nets, views), lrate=LRATE, lrate_decay=DECAY, use_graph=use_graph)


def _state(tr, losses=()):
    torch.cuda.synchronize()
    return [tr.flat_p.clone(), tr.m.clone(), tr.v.clone(), tr.state.clone(), torch.cat([l.reshape(1) for l in losses]) if losses else tr.state[:1].clone()]


def _rays(G, n, seed):
    sb = G.synth.ray_batch("lego", n, seed=seed)
    return G.dev(sb["rays"]), G.dev(np.random.default_rng(seed).random((n, 3), dtype=np.float32))


def _copy_from(dst, src):
    with torch.no_grad():
        for a, b in ((dst.flat_p, src.flat_p), (dst.m, src.m), (dst.v, src.v), (dst.state, src.state)):
            a.copy_(b)


# ---- a short step is a step of that size --------------------------------------------------------------------------------------

SHORT_CASES = [(v, g, mode) for v in (True, False) for g, mode in ((True, "rays"), (False, "rays"), (True, "pixels"))]


@pytest.mark.parametrize("views,use_graph,mode", SHORT_CASES,
                         ids=[f"{'views' if v else 'noviews'}-{'graph' if g else 'eager'}-{m}" for v, g, m in SHORT_CASES])
def test_short_step_is_a_step_of_that_size(G, views, use_graph, mode):
    """A FusedTrainStep built for 1024 rays, after one full step, and one built for 816 rays with its parameters, moments, state
    and generator state: one step on the same 816 rays (or the same 816 pixels of one pose) gives the same bits"""
    big = _step(G, views, CAP, use_graph)
    rays, target = _rays(G, CAP, seed=1)
    big.rays.copy_(rays); big.target.copy_(target)
    big.step_device()
    small = _step(G, views, SHORT, use_graph)
    _copy_from(small, big)
    rays, target = _rays(G, SHORT, seed=2)
    H, W, _, c2w = G.synth.lego_camera(400)
    pix = torch.randperm(H * W, device=G.DEV)[:SHORT]
    for tr in (big, small):
        tr.rays[:, :SHORT].copy_(rays); tr.target[:SHORT].copy_(target)
    torch.manual_seed(3)
    rng = torch.cuda.get_rng_state()
    runs = []
    for tr in (big, small):
        torch.cuda.set_rng_state(rng)
        if mode == "rays":
            tr.step_device(n_rays=SHORT) if tr is big else tr.step_device()
        else:
            tr.step_device(c2w=torch.from_numpy(c2w), pixel_index=pix)
        runs.append(_state(tr) + [torch.cuda.get_rng_state()])
    a, b = runs
    assert float(a[3][1]) == 2 and np.isfinite(float(a[3][0]))
    assert_same_bits(a[:5], b[:5], f"{CAP}-ray step at {SHORT} rays vs a {SHORT}-ray step")
    assert torch.equal(a[5], b[5]), "the generator advanced differently"
    if use_graph:
        assert sorted(big._graphs) == [SHORT, CAP]


# ---- an epoch with a short tail ------------------------------------------------------------------------------------------------

def _epoch_data(G):
    """3 x 1024 + 816 shuffled rays_rgb of four 32 x 32 views of the lego camera, with random colours"""
    H, W, K, _ = G.synth.lego_camera(32)
    rng = np.random.default_rng(0)
    poses = np.stack([G.synth.pose_spherical(90.0 * i, -30.0, 4.0) for i in range(4)], 0)
    images = rng.random((4, H, W, 3), dtype=np.float32)
    rays = np.stack([np.stack(G.synth.camera_rays(H, W, K, p[:3, :4]), 0) for p in poses], 0)
    rays_rgb = np.concatenate([rays, images[:, None]], 1).transpose(0, 2, 3, 1, 4).reshape(-1, 3, 3).astype(np.float32)
    rays_rgb = rays_rgb[rng.permutation(rays_rgb.shape[0])[:3 * CAP + SHORT]]
    return H, W, K, images, poses, rays_rgb


def _fused_epochs(G, views, steps, use_graph):
    H, W, K, images, poses, rays_rgb = _epoch_data(G)
    tr = _step(G, views, CAP, use_graph)
    torch.manual_seed(0)
    batcher = G.nb.DeviceRayBatcher(images, poses, H, W, CAP, rays_rgb=rays_rgb, device=G.DEV)
    losses, sizes = [], []
    for _ in range(steps):
        batch_rays, target = batcher.next()
        n = target.shape[0]
        tr.rays[:, :n].copy_(batch_rays); tr.target[:n].copy_(target)
        tr.step_device(n_rays=n)
        losses.append(tr.state[0:1].clone())
        sizes.append(n)
    return _state(tr, losses), sizes, tr


@pytest.mark.parametrize("views", [True, False], ids=["views", "noviews"])
def test_epochs_with_a_short_tail(G, views):
    """DeviceRayBatcher over 3 x 1024 + 816 rays through two epoch ends: graph replays give the bits of the eager step, and the
    trajectory is that of the drop-in loop (render + 2 x img2mse + backward + torch.optim.Adam + the host decay, run_nerf.py:760-784)
    on the same batches and draws"""
    steps = 9
    graph, sizes, tr = _fused_epochs(G, views, steps, True)
    eager, sizes_e, _ = _fused_epochs(G, views, steps, False)
    assert sizes == sizes_e == [CAP, CAP, CAP, SHORT, CAP, CAP, CAP, SHORT, CAP]
    assert float(graph[3][1]) == steps and np.all(np.isfinite(graph[4].cpu().numpy()))
    assert_same_bits(graph, eager, "graph vs eager")
    # the drop-in loop
    H, W, K, images, poses, rays_rgb = _epoch_data(G)
    nets = _nets(G, views)
    init = torch.cat([p.detach().reshape(-1) for n in nets for p in n.parameters()])
    kw = _kwargs(G, nets, views)
    opt = torch.optim.Adam([p for n in nets for p in n.parameters()], lr=LRATE, betas=(0.9, 0.999))
    torch.manual_seed(0)
    batcher = G.nb.DeviceRayBatcher(images, poses, H, W, CAP, rays_rgb=rays_rgb, device=G.DEV)
    losses = []
    for global_step in range(steps):
        batch_rays, target = batcher.next()
        rgb, _, _, ex = G.nb.render(H, W, K, chunk=32768, rays=batch_rays, retraw=True, **kw)
        opt.zero_grad()
        loss = G.nb.img2mse(rgb, target) + G.nb.img2mse(ex["rgb0"], target)
        loss.backward()
        opt.step()
        for pg in opt.param_groups:
            pg["lr"] = LRATE * (0.1 ** (global_step / (DECAY * 1000)))
        losses.append(float(loss.detach()))
    fused = graph[4].cpu().numpy()
    assert np.allclose(losses, fused, rtol=2e-4), (losses, fused.tolist())
    worst, off = 0.0, 0
    for p in [p for n in nets for p in n.parameters()]:
        k = p.numel()
        da = (p.detach().reshape(-1) - init[off:off + k]).cpu().numpy()
        db = (graph[0][off:off + k] - init[off:off + k]).cpu().numpy()
        worst = max(worst, rel_l2(db, da))
        off += k
    print(f"[variable batch] views={views}: losses {fused.tolist()}; worst parameter-update rel-L2 vs drop-in {worst:.3e}")
    assert worst < 5e-2, worst


# ---- resume across the short batch ---------------------------------------------------------------------------------------------

def _resumable(G, views, steps, tmp_path, save_after=None, resume=None):
    """`steps` steps of the batching loop of INTEGRATION §5a; save after `save_after` of them, or start from the file `resume`
    -> [flat_p, m, v, state, losses]"""
    H, W, K, images, poses, rays_rgb = _epoch_data(G)
    nets = _nets(G, views)
    ck = None
    if resume is not None:
        ck = torch.load(resume, map_location=G.DEV)
        for n, sd in zip(nets, ck["nets"]):
            n.load_state_dict(sd)
    tr = _step(G, views, CAP, True, nets=nets)
    torch.manual_seed(0)
    batcher = G.nb.DeviceRayBatcher(images, poses, H, W, CAP, rays_rgb=rays_rgb, device=G.DEV)
    if ck is not None:
        tr.load_state_dict(ck["train_step"])
        batcher.load_state_dict(ck["batcher"])
    losses = []
    for i in range(steps):
        batch_rays, target = batcher.next()
        n = target.shape[0]
        tr.rays[:, :n].copy_(batch_rays); tr.target[:n].copy_(target)
        tr.step_device(n_rays=n)
        losses.append(tr.state[0:1].clone())
        if save_after == i + 1:
            path = str(tmp_path / "ck.tar")
            torch.save({"nets": [n_.state_dict() for n_ in nets], "train_step": tr.state_dict(), "batcher": batcher.state_dict()}, path)
    return _state(tr, losses)


@pytest.mark.parametrize("views", [True, False], ids=["views", "noviews"])
@pytest.mark.parametrize("k", [3, 4], ids=["before_short", "after_short"])
def test_resume_across_the_short_batch(G, tmp_path, views, k):
    """Interrupted after step 3 (the next step is the first short one) or after step 4 (the short step is behind it, and the
    resumed step has not captured 816 rays yet: it does so at step 8, the uninterrupted run at step 4), resumed in a new step
    object: the same bits as the uninterrupted 8 steps.  The lazy capture leaves the generator untouched."""
    whole = _resumable(G, views, 8, tmp_path / "whole")
    (tmp_path / "first").mkdir()
    first = _resumable(G, views, k, tmp_path / "first", save_after=k)
    second = _resumable(G, views, 8 - k, tmp_path, resume=str(tmp_path / "first" / "ck.tar"))
    assert float(whole[3][1]) == 8
    assert_same_bits(whole, second[:4] + [torch.cat([first[4], second[4]])], f"resumed after {k} steps")


# ---- memory ---------------------------------------------------------------------------------------------------------------------

BUFS = ("act_c", "mask_c", "act_f", "mask_f", "ws", "bws")


def _needs(G, tr, n):
    """the bytes the library's size queries ask for an n-ray step, per buffer"""
    lib, Sc, Sf = tr.lib, tr.Sc, tr.Sc + tr.Ni
    out = {}
    for tag, S, np_ in (("c", Sc, tr._np_c), ("f", Sf, tr._np_f)):
        ab, mb = C.c_size_t(0), C.c_size_t(0)
        assert lib.nerf_b200_train_record_bytes(n, S, C.byref(np_), C.byref(ab), C.byref(mb)) == 0
        out["act_" + tag], out["mask_" + tag] = ab.value, mb.value
    out["ws"] = lib.nerf_b200_march_workspace_bytes(n, Sf)
    out["bws"] = lib.nerf_b200_render_rays_bwd_tc_workspace_bytes(n, Sc, C.byref(tr._np_c), Sf, C.byref(tr._np_f)) + 1024
    return out


def test_new_sizes_allocate_nothing(G):
    """Steps at 1024, 816 and 1 rays run on the capacity's records and workspaces (their size queries fit there): the same
    data_ptrs, and torch.cuda.memory_allocated() unchanged by the two captures.  The full-size step is not disturbed by them:
    it gives the bits of a step object that never saw another size."""
    tr = _step(G, True, CAP)
    ref = _step(G, True, CAP)
    cap = {k: (tr._sized[CAP][k].data_ptr(), tr._sized[CAP][k].numel()) for k in BUFS}
    rays, target = _rays(G, CAP, seed=4)
    for t in (tr, ref):
        t.rays.copy_(rays); t.target.copy_(target)
    mem = {}
    for n in (CAP, SHORT, 1):
        need = _needs(G, tr, n)
        tr.step_device(n_rays=n)
        torch.cuda.synchronize()
        mem[n] = torch.cuda.memory_allocated()
        for k in BUFS:
            if need[k] <= cap[k][1]:
                assert tr._sized[n][k].data_ptr() == cap[k][0], (n, k)
        assert np.isfinite(float(tr.state[0]))
    print(f"[variable batch] torch.cuda.memory_allocated() after steps at {list(mem)} rays: {list(mem.values())} bytes")
    assert mem[SHORT] == mem[CAP] and mem[1] == mem[CAP], mem
    assert sorted(tr._graphs) == [1, SHORT, CAP]
    # the capacity's graph after the other captures: the bits of `ref`, given the same state and draws
    _copy_from(ref, tr)
    torch.manual_seed(5)
    rng = torch.cuda.get_rng_state()
    runs = []
    for t in (tr, ref):
        torch.cuda.set_rng_state(rng)
        t.step_device()
        runs.append(_state(t))
    assert_same_bits(runs[0], runs[1], "full-size step after captures at 816 and 1 rays")


def test_a_size_whose_plan_needs_more_records_gets_its_own(G):
    """The library's tile plan does not shrink with n everywhere: for some n < 1024 the records or workspaces need more than at
    1024.  Such a size gets buffers of its own (the capacity's stay as they were) and still takes the step of a FusedTrainStep
    built for n rays"""
    tr = _step(G, True, CAP)
    have = {k: tr._sized[CAP][k].numel() for k in BUFS}
    grow = next((n for n in range(CAP - 1, 0, -1) if any(v > have[k] for k, v in _needs(G, tr, n).items())), None)
    assert grow is not None, "no size below 1024 needs more than the capacity on this GPU"
    cap_ptrs = {k: tr._sized[CAP][k].data_ptr() for k in BUFS}
    rays, target = _rays(G, grow, seed=6)
    tr.rays[:, :grow].copy_(rays); tr.target[:grow].copy_(target)
    small = _step(G, True, grow)
    small.rays.copy_(rays); small.target.copy_(target)
    torch.manual_seed(7)
    rng = torch.cuda.get_rng_state()
    runs = []
    for t in (tr, small):
        torch.cuda.set_rng_state(rng)
        t.step_device(n_rays=grow)
        runs.append(_state(t))
    need = _needs(G, tr, grow)
    grown = [k for k in BUFS if need[k] > have[k]]
    print(f"[variable batch] {grow} rays need more than {CAP} in {grown}: " + ", ".join(f"{k} {need[k]} > {have[k]}" for k in grown))
    assert all(tr._sized[grow][k].numel() >= need[k] for k in BUFS)
    assert all(tr._sized[grow][k].data_ptr() != cap_ptrs[k] for k in grown)
    assert {k: tr._sized[CAP][k].data_ptr() for k in BUFS} == cap_ptrs
    assert_same_bits(runs[0], runs[1], f"{CAP}-ray step at {grow} rays vs a {grow}-ray step")


# ---- refusals -------------------------------------------------------------------------------------------------------------------

def test_refusals_launch_nothing_and_change_nothing(G):
    tr = _step(G, True, CAP)
    rays, target = _rays(G, CAP, seed=8)
    tr.rays.copy_(rays); tr.target.copy_(target)
    tr.step_device()
    before, rng, l0 = _state(tr), torch.cuda.get_rng_state(), G.nb.launch_count()
    rh, th = rays.cpu(), target.cpu()
    rh_big = torch.cat([rh, rh[:, :1]], 1)
    pix = torch.arange(SHORT, device=G.DEV)
    c2w = torch.from_numpy(G.synth.lego_camera(400)[3])
    bad = {
        "n_rays=0": lambda: tr.step_device(n_rays=0),
        "n_rays>capacity": lambda: tr.step_device(n_rays=CAP + 1),
        "pixel_index>capacity": lambda: tr.step_device(c2w=c2w, pixel_index=torch.arange(CAP + 1, device=G.DEV)),
        "pixel_index != n_rays": lambda: tr.step_device(c2w=c2w, pixel_index=pix, n_rays=SHORT - 1),
        "call: n=0": lambda: tr(rh[:, :0], th[:0]),
        "call: n>capacity": lambda: tr(rh_big, torch.cat([th, th[:1]])),
        "call: target rows differ": lambda: tr(rh[:, :SHORT], th[:SHORT - 1]),
        "call: target width": lambda: tr(rh[:, :SHORT], torch.zeros(SHORT, 4)),
        "call: rays shape": lambda: tr(rh[:1, :SHORT], th[:SHORT]),
    }
    for what, call in bad.items():
        with pytest.raises(RuntimeError):
            call()
        assert G.nb.launch_count() == l0, what
    torch.cuda.synchronize()
    assert_same_bits(before, _state(tr), "after the refusals")
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    assert sorted(tr._graphs) == [CAP] and sorted(tr._sized) == [CAP]


# ---- GraphedRender -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("views", [True, False], ids=["views", "noviews"])
def test_graphed_render_renders_a_frame_with_a_tail_chunk(G, views):
    """A 400 x 400 frame = 39 x 4096 + 256 rays through GraphedRender(n_rays=4096) in 40 calls: the bits of eager render() with
    chunk=4096 on the same rays.  The 256-ray tail is captured once; a second frame adds no graph."""
    H, W, K, c2w = G.synth.lego_camera(400)
    o, d = G.synth.camera_rays(H, W, K, c2w)
    rays_h = torch.from_numpy(np.stack([o.reshape(-1, 3), d.reshape(-1, 3)], 0)).pin_memory()
    kw = _kwargs(G, _nets(G, views), views)
    kw.update(perturb=0., raw_noise_std=0.)
    with torch.no_grad():
        rgb, disp, acc, _ = G.nb.render(H, W, K, chunk=4096, rays=rays_h.to(G.DEV), **kw)
    want = torch.cat([rgb.reshape(-1, 3), disp.reshape(-1, 1), acc.reshape(-1, 1)], 1).cpu()
    g = G.nb.GraphedRender(H, W, K, 4096, **kw)
    for frame in range(2):
        outs = []
        for i in range(0, H * W, 4096):
            out = g(rays_h[:, i:i + 4096])
            outs.append(out.clone())
        assert [x.shape[0] for x in outs] == [4096] * 39 + [256]
        assert g.device_out[0].shape == (256, 3)
        got = torch.cat(outs)
        assert torch.equal(bits(got), bits(want)), f"frame {frame}: {int((bits(got) != bits(want)).any(1).sum())} rays differ"
        assert sorted(g._graphs) == [256, 4096]
    for bad in (rays_h[:, :0], rays_h[:, :4097], rays_h[:1, :16]):
        with pytest.raises(RuntimeError):
            g(bad)
    assert sorted(g._graphs) == [256, 4096]
