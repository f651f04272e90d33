"""Resuming FusedTrainStep training from a checkpoint.  A run interrupted after k steps, saved with torch.save, dropped and
rebuilt through create_nerf continues to the same bits as the run that was never interrupted (parameters, Adam moments, step
state, every loss), with the device draws of perturb = 1 and raw_noise_std > 0 on.  A checkpoint of the reference's format
written by the drop-in loop continues on the fused step, and a fused checkpoint reloads in the unmodified reference."""
import argparse
import gc
import os
import sys
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu
LRATE, DECAY = 5e-4, 0.002                      # decay_steps = 2: a step count off by one changes the rate visibly


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


def _args(tmp, views=True, ft_path=None):
    """create_nerf's arguments (run_nerf.py config_parser) for a blender-type scene"""
    os.makedirs(os.path.join(tmp, "e"), exist_ok=True)
    return argparse.Namespace(multires=10, multires_views=4, i_embed=0, use_viewdirs=views, N_importance=64, N_samples=64, netdepth=8,
                              netwidth=256, netdepth_fine=8, netwidth_fine=256, netchunk=65536, lrate=LRATE, basedir=str(tmp), expname="e",
                              ft_path=ft_path, no_reload=ft_path is None, perturb=1.0, white_bkgd=True, raw_noise_std=1.0,
                              dataset_type="blender", no_ndc=False, lindisp=False)


def _save(path, tr, kw, opt, batcher=None):
    """the reference's checkpoint dict (run_nerf.py:794-799) plus the continuation state under trainer.RESUME_KEY"""
    from nerf_pytorch_b200.trainer import RESUME_KEY
    tr.attach_optimizer(opt)
    extra = {"train_step": tr.state_dict()}
    if batcher is not None:
        extra["batcher"] = batcher.state_dict()
    torch.save({"global_step": tr.global_step, "network_fn_state_dict": kw["network_fn"].state_dict(),
                "network_fine_state_dict": kw["network_fine"].state_dict(), "optimizer_state_dict": opt.state_dict(), RESUME_KEY: extra}, path)


# ---- bitwise continuation ----------------------------------------------------------------------------------------------------

@dataclass
class Case:
    name: str
    batching: bool          # shuffled rays_rgb (use_batching) or random pixels of one image per step (no_batching)
    B: int                  # rays per step
    n_img: int
    res: int
    views: bool = True
    use_graph: bool = True
    k: int = 4              # steps before the interruption, and after it


CASES = [
    Case("rays_graph", True, 1024, 12, 16),                         # 3 batches per epoch: epoch ends after steps 3 and 6
    Case("rays_eager", True, 1024, 12, 16, use_graph=False),
    Case("pixels_precrop", False, 1024, 5, 40),                     # precrop_iters = 6 > k
    Case("noviews", True, 1024, 12, 16, views=False),
    Case("rays_4096", True, 4096, 12, 32),
]


def _data(G, c):
    H, W, K, _ = G.synth.lego_camera(c.res)
    rng = np.random.default_rng(0)
    images = rng.random((c.n_img, H, W, 3), dtype=np.float32)
    poses = np.stack([G.synth.pose_spherical(360.0 * i / c.n_img, -30.0, 4.0) for i in range(c.n_img)], 0)
    if not c.batching:
        return H, W, K, dict(images=images, poses=poses, i_train=list(range(1, c.n_img)), precrop_iters=6, precrop_frac=0.5)
    rays = np.stack([np.stack(G.synth.camera_rays(H, W, K, p[:3, :4]), 0) for p in poses], 0)
    rays_rgb = np.concatenate([rays, images[:, None]], 1).transpose(0, 2, 3, 1, 4).reshape(-1, 3, 3).astype(np.float32)
    rays_rgb = rays_rgb[rng.permutation(rays_rgb.shape[0])]         # run_nerf.py:688
    assert rays_rgb.shape[0] == 3 * c.B
    return H, W, K, dict(images=images, poses=poses, rays_rgb=rays_rgb)


def _train(G, tmp, c, steps, resume_from=None, save_to=None, seed=0):
    """`steps` steps of the fused loop: a fresh run, or one rebuilt from the checkpoint `resume_from` as INTEGRATION §5a does
    -> [flat parameters, m, v, state, losses]"""
    from nerf_pytorch_b200 import api
    from nerf_pytorch_b200.trainer import RESUME_KEY, FusedTrainStep
    H, W, K, data = _data(G, c)
    torch.manual_seed(seed)
    kw, _, start, _, opt = api.create_nerf(_args(tmp, c.views, resume_from), device=G.DEV)
    kw.update(near=2., far=6.)
    tr = FusedTrainStep(H, W, K, c.B, kw, lrate=LRATE, lrate_decay=DECAY, use_graph=c.use_graph)
    tr.load_optimizer(opt)
    batcher = G.nb.DeviceRayBatcher(data.pop("images"), data.pop("poses"), H, W, c.B, device=G.DEV, **data)
    if resume_from is not None:
        extra = torch.load(resume_from, map_location=G.DEV)[RESUME_KEY]
        tr.load_state_dict(extra["train_step"])
        batcher.load_state_dict(extra["batcher"])
        assert start == tr.global_step == c.k
    losses = []
    for _ in range(steps):
        if c.batching:
            batch_rays, target = batcher.next()
            tr.rays.copy_(batch_rays)
            tr.target.copy_(target)
            tr.step_device()
        else:
            c2w, pix, target = batcher.next()
            tr.target.copy_(target)
            tr.step_device(c2w=c2w, pixel_index=pix)
        losses.append(tr.state[0:1].clone())
    if save_to is not None:
        _save(save_to, tr, kw, opt, batcher)
    torch.cuda.synchronize()
    return [tr.flat_p.clone(), tr.m.clone(), tr.v.clone(), tr.state.clone(), torch.cat(losses)]


@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_interrupted_run_continues_bitwise(G, tmp_path, c):
    whole = _train(G, tmp_path / "whole", c, 2 * c.k)
    path = str(tmp_path / "first" / "e" / f"{c.k:06d}.tar")
    first = _train(G, tmp_path / "first", c, c.k, save_to=path)
    gc.collect()                                                    # nets, step, graph and batcher of the first half are gone
    second = _train(G, tmp_path / "second", c, c.k, resume_from=path, seed=123)
    assert np.all(np.isfinite(whole[4].cpu().numpy()))
    assert float(whole[3][1]) == 2 * c.k
    assert_same_bits(whole, second[:4] + [torch.cat([first[4], second[4]])], c.name)


# ---- load_optimizer -------------------------------------------------------------------------------------------------------

def _kwargs(G, nets, perturb=1., noise=1.):
    return dict(network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64, N_importance=64, perturb=perturb,
                white_bkgd=True, raw_noise_std=noise, use_viewdirs=True, ndc=False, lindisp=False, near=2., far=6.)


def _batch(G, N, seed=8):
    sb = G.synth.ray_batch("lego", N, seed=seed)
    tgt = np.random.default_rng(2).random((N, 3), dtype=np.float32)
    return sb, torch.from_numpy(sb["rays"]).pin_memory(), torch.from_numpy(tgt).pin_memory()


def test_empty_optimizer_changes_nothing(G):
    """load_optimizer on an optimizer without state: the same bits as not calling it, and the same library launches per step (one
    ray packing outside the graph; the rest is the captured graph)"""
    from nerf_pytorch_b200.trainer import FusedTrainStep
    N = 1024
    sb, rays_h, tgt_h = _batch(G, N)
    runs, launches = [], []
    for call in (False, True):
        nets = [G.make_net(G.synth.nerf_state(0)), G.make_net(G.synth.nerf_state(1))]
        torch.manual_seed(9)
        tr = FusedTrainStep(400, 400, sb["K"], N, _kwargs(G, nets), lrate=LRATE, lrate_decay=DECAY)
        if call:
            opt = torch.optim.Adam([p for n in nets for p in n.parameters()], lr=LRATE)
            assert tr.load_optimizer(opt) is opt and len(opt.state) == 48
        l0 = G.nb.launch_count()
        losses = torch.tensor([tr(rays_h, tgt_h) for _ in range(5)])
        launches.append(G.nb.launch_count() - l0)
        runs.append([tr.flat_p.clone(), tr.m.clone(), tr.v.clone(), tr.state.clone(), losses])
    assert_same_bits(runs[0], runs[1], "load_optimizer(empty)")
    assert launches[0] == launches[1], launches


@pytest.mark.parametrize("shared", [False, True])
def test_optimizer_round_trip(G, shared):
    """attach_optimizer -> optimizer.state_dict() -> a new optimizer over new networks -> load_optimizer: the moments and the step
    count are the same bits, and the new optimizer's state aliases the new step's flat moments.  A fine net shared with the coarse
    one (network_fine=None) counts once."""
    from nerf_pytorch_b200.trainer import FusedTrainStep
    N = 1024
    sb, rays_h, tgt_h = _batch(G, N)

    def nets():
        n = [G.make_net(G.synth.nerf_state(0)), G.make_net(G.synth.nerf_state(1))]
        return [n[0], None] if shared else n
    na = nets()
    tr_a = FusedTrainStep(400, 400, sb["K"], N, _kwargs(G, na), lrate=LRATE, lrate_decay=DECAY)
    for _ in range(3):
        tr_a(rays_h, tgt_h)
    opt_a = tr_a.attach_optimizer(torch.optim.Adam(tr_a.params, lr=LRATE))
    sd = opt_a.state_dict()
    assert len(sd["state"]) == (24 if shared else 48)
    nb_ = nets()
    for a, b in zip(na, nb_):
        if a is not None:
            b.load_state_dict(a.state_dict())
    params_b = [p for n in nb_ if n is not None for p in n.parameters()]
    opt_b = torch.optim.Adam(params_b, lr=LRATE)
    opt_b.load_state_dict(sd)
    tr_b = FusedTrainStep(400, 400, sb["K"], N, _kwargs(G, nb_), lrate=LRATE, lrate_decay=DECAY)
    tr_b.load_optimizer(opt_b)
    torch.cuda.synchronize()
    assert tr_b.global_step == 3
    for x, y in ((tr_a.m, tr_b.m), (tr_a.v, tr_b.v), (tr_a.flat_p, tr_b.flat_p)):
        assert torch.equal(bits(x), bits(y))
    lo, hi = tr_b.m.data_ptr(), tr_b.m.data_ptr() + 4 * tr_b.m.numel()
    assert all(lo <= opt_b.state[p]["exp_avg"].data_ptr() < hi for p in params_b)
    assert abs(opt_b.param_groups[0]["lr"] - LRATE * 0.1 ** (2 / (DECAY * 1000))) < 1e-12


# ---- interoperation with the reference's loop -----------------------------------------------------------------------------

def test_reference_checkpoint_continues_on_the_fused_step(G, tmp_path):
    """The drop-in loop (render + img2mse + backward + torch.optim.Adam + the host decay, run_nerf.py:760-784) runs k steps and
    saves as the reference does; FusedTrainStep.load_optimizer continues from that file and follows the drop-in loop's own
    next steps within test_gpu_trainer.py's gates.  Its first step uses the rate the reference would."""
    from nerf_pytorch_b200 import api
    from nerf_pytorch_b200.trainer import FusedTrainStep
    N, k, j = 1024, 4, 4
    sb, rays_h, tgt_h = _batch(G, N)
    rays, target = rays_h.to(G.DEV), tgt_h.to(G.DEV)
    torch.manual_seed(0)
    kw, _, _, grad_vars, opt = api.create_nerf(_args(tmp_path), device=G.DEV)
    kw.update(near=2., far=6.)

    def dropin_steps(n, global_step):
        losses = []
        for _ in range(n):
            rgb, _, _, ex = G.nb.render(400, 400, sb["K"], chunk=32768, rays=rays, retraw=True, **kw)
            opt.zero_grad()
            loss = G.nb.img2mse(rgb, target) + G.nb.img2mse(ex["rgb0"], target)
            loss.backward()
            opt.step()
            for pg in opt.param_groups:
                pg["lr"] = LRATE * (0.1 ** (global_step / (DECAY * 1000)))
            global_step += 1
            losses.append(float(loss.detach()))
        return losses
    dropin_steps(k, 0)
    path = str(tmp_path / "e" / f"{k:06d}.tar")
    torch.save({"global_step": k - 1,                            # saved before its increment (run_nerf.py:794, :872)
                "network_fn_state_dict": kw["network_fn"].state_dict(), "network_fine_state_dict": kw["network_fine"].state_dict(),
                "optimizer_state_dict": opt.state_dict()}, path)
    rng, rate_next = torch.cuda.get_rng_state(), opt.param_groups[0]["lr"]
    at_k = [p.detach().clone() for p in grad_vars]
    losses_a = dropin_steps(j, k)
    after_a = [p.detach().clone() for p in grad_vars]
    torch.manual_seed(7)
    kw_b, _, start, grad_vars_b, opt_b = api.create_nerf(_args(tmp_path, ft_path=path), device=G.DEV)
    kw_b.update(near=2., far=6.)
    assert start == k - 1
    tr = FusedTrainStep(400, 400, sb["K"], N, kw_b, lrate=LRATE, lrate_decay=DECAY)
    tr.load_optimizer(opt_b)
    assert tr.global_step == k                                  # Adam's step count, not the file's global_step
    torch.cuda.set_rng_state(rng)                               # the draws the drop-in loop made after the save
    losses_b = []
    for i in range(j):
        losses_b.append(tr(rays_h, tgt_h))
        if i == 0:
            rate = float(tr.state[2])
    assert abs(rate - rate_next) <= 1e-6 * rate_next, (rate, rate_next)
    assert np.allclose(losses_a, losses_b, rtol=2e-4), (losses_a, losses_b)
    worst = max(rel_l2((pb.detach() - p0).cpu().numpy(), (pa - p0).cpu().numpy()) for pa, pb, p0 in zip(after_a, grad_vars_b, at_k))
    assert worst < 5e-2, worst


def test_fused_checkpoint_reloads_in_the_reference(G, tmp_path):
    """attach_optimizer, then the reference's save: the unmodified reference's create_nerf (run_nerf.py:215-233) reloads the file
    with the step's global_step as `start`, its moments and step count in Adam and its weights in both nets"""
    import ref_gpu
    if not ref_gpu.available():
        pytest.skip("oracle/_ref missing (built by __graft_entry__.build() where the reference checkout exists)")
    from nerf_pytorch_b200 import api
    from nerf_pytorch_b200.trainer import FusedTrainStep
    N, k = 1024, 3
    sb, rays_h, tgt_h = _batch(G, N)
    torch.manual_seed(0)
    kw, _, _, _, opt = api.create_nerf(_args(tmp_path), device=G.DEV)
    kw.update(near=2., far=6.)
    tr = FusedTrainStep(400, 400, sb["K"], N, kw, lrate=LRATE, lrate_decay=DECAY)
    tr.load_optimizer(opt)
    for _ in range(k):
        tr(rays_h, tgt_h)
    path = str(tmp_path / "e" / f"{k:06d}.tar")
    _save(path, tr, kw, opt)
    torch.cuda.synchronize()
    before = set(sys.modules)
    try:
        ref = ref_gpu.load("run_nerf_ref_resume")
        kw_r, _, start, grad_vars_r, opt_r = ref.create_nerf(_args(tmp_path, ft_path=path))
    finally:
        # ref_gpu.load imports the reference's modules against empty imageio / configargparse stand-ins; forget them, so that
        # a later import of the reference (test_gpu_dropin.py's, with working stand-ins) does not pick them up
        for name in set(sys.modules) - before:
            if name in ("imageio", "matplotlib", "matplotlib.pyplot", "configargparse") or \
                    str(getattr(sys.modules[name], "__file__", "")).startswith(ref_gpu.REF):
                del sys.modules[name]
    assert start == k
    assert not isinstance(kw_r["network_fn"], G.nb.NeRF)
    assert len(grad_vars_r) == len(tr.params) == 48
    off = 0
    for p, q in zip(tr.params, grad_vars_r):
        n = p.numel()
        st = opt_r.state[q]
        assert float(st["step"]) == k
        assert torch.equal(bits(q), bits(p)), "weights"
        assert torch.equal(bits(st["exp_avg"].reshape(-1)), bits(tr.m[off:off + n])), "exp_avg"
        assert torch.equal(bits(st["exp_avg_sq"].reshape(-1)), bits(tr.v[off:off + n])), "exp_avg_sq"
        off += n
    assert abs(opt_r.param_groups[0]["lr"] - LRATE * 0.1 ** ((k - 1) / (DECAY * 1000))) < 1e-12
