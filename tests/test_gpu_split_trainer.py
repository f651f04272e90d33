"""FusedTrainStep on precision tc_split with set_backward('tc_split'): the split training image, split records and split backward
inside the step's CUDA graph.

(a) its gradient is the autograd split path's, bit for bit, given the same seeds;
(b) its steps follow torch.optim.Adam on the drop-in split step (as tests/test_gpu_trainer.py does for tc_fp16);
(c) the same bits run to run, a short step of n < N rays has the bits of a step built for n, and a state_dict round trip
    continues bit for bit."""
import numpy as np
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


@pytest.fixture
def split(G):
    G.nb.set_precision("tc_split")
    G.nb.set_backward("tc_split")
    yield
    G.nb.set_precision("tc_fp16")
    G.nb.set_backward("tc")


def _kwargs(G, nets):
    return dict(network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64, N_importance=128, perturb=0.,
                white_bkgd=True, raw_noise_std=0., use_viewdirs=True, ndc=False, lindisp=False, near=2., far=6.)


def _nets(G):
    return [G.make_net(G.synth.nerf_state(0)), G.make_net(G.synth.nerf_state(1))]


def _batch(G, N, seed=8):
    sb = G.synth.ray_batch("lego", N, seed=seed)
    return sb, G.dev(sb["rays"]), G.dev(np.random.default_rng(2).random((N, 3), dtype=np.float32))


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def test_refusal_without_the_split_backward(G, split):
    from nerf_pytorch_b200.trainer import FusedTrainStep
    G.nb.set_backward("exact")
    sb, _, _ = _batch(G, 64)
    with pytest.raises(RuntimeError, match="tc_fp16"):
        FusedTrainStep(400, 400, sb["K"], 64, _kwargs(G, _nets(G)))


def test_gradient_is_the_autograd_split_paths(G, split):
    from nerf_pytorch_b200.trainer import FusedTrainStep
    N = 300
    sb, rays, target = _batch(G, N)
    tr = FusedTrainStep(400, 400, sb["K"], N, _kwargs(G, _nets(G)), use_graph=False)
    tr.rays[:, :N].copy_(rays); tr.target[:N].copy_(target)
    tr._pack_rays(n=N); tr._fwd_bwd(N)
    torch.cuda.synchronize()
    nets_a = _nets(G)
    rgb, _, _, ex = G.nb.render(400, 400, sb["K"], chunk=32768, rays=rays, retraw=True, **_kwargs(G, nets_a))
    assert torch.equal(_bits(rgb), _bits(tr.out["rgb"][:N])) and torch.equal(_bits(ex["rgb0"]), _bits(tr.out["rgb0"][:N]))
    torch.autograd.backward([rgb, ex["rgb0"]], [tr.out["g_rgb"][:N].clone(), tr.out["g_rgb0"][:N].clone()])
    for pa, pb in zip([p for n in nets_a for p in n.parameters()], tr.params):
        assert torch.equal(_bits(pa.grad), _bits(pb.grad))


def test_steps_follow_autograd_adam(G, split):
    from nerf_pytorch_b200.trainer import FusedTrainStep
    N, steps, lrate, decay = 200, 4, 5e-4, 0.002
    sb, rays, target = _batch(G, N)
    nets_a = _nets(G)
    opt = torch.optim.Adam([p for n in nets_a for p in n.parameters()], lr=lrate, betas=(0.9, 0.999))
    losses_a = []
    for step in range(steps):
        rgb, _, _, ex = G.nb.render(400, 400, sb["K"], chunk=32768, rays=rays, retraw=True, **_kwargs(G, nets_a))
        opt.zero_grad()
        loss = G.nb.img2mse(rgb, target) + G.nb.img2mse(ex["rgb0"], target)
        loss.backward()
        opt.step()
        for pg in opt.param_groups:
            pg["lr"] = lrate * (0.1 ** (step / (decay * 1000)))
        losses_a.append(float(loss.detach()))
    nets_b = _nets(G)
    init = [p.detach().clone() for n in nets_b for p in n.parameters()]
    tr = FusedTrainStep(400, 400, sb["K"], N, _kwargs(G, nets_b), lrate=lrate, lrate_decay=decay)
    rays_h, tgt_h = rays.cpu().pin_memory(), target.cpu().pin_memory()
    losses_b = [tr(rays_h, tgt_h) for _ in range(steps)]
    assert tr.global_step == steps
    assert np.allclose(losses_a, losses_b, rtol=2e-4), (losses_a, losses_b)
    worst = max(rel_l2((pb.detach() - p0).cpu().numpy(), (pa.detach() - p0).cpu().numpy())
                for pa, pb, p0 in zip([p for n in nets_a for p in n.parameters()], tr.params, init))
    assert worst < 5e-2, worst


def test_bits_run_to_run_short_steps_and_resume(G, split):
    from nerf_pytorch_b200.trainer import FusedTrainStep
    N, n = 256, 200
    sb, rays, target = _batch(G, N, seed=3)
    rays_h, tgt_h = rays.cpu().pin_memory(), target.cpu().pin_memory()

    def run(cap, k, steps):
        tr = FusedTrainStep(400, 400, sb["K"], cap, _kwargs(G, _nets(G)))
        for _ in range(steps):
            tr(rays_h[:, :k], tgt_h[:k])
        return tr
    a, b = run(N, N, 2), run(N, N, 2)
    assert torch.equal(_bits(a.flat_p), _bits(b.flat_p)) and torch.equal(_bits(a.m), _bits(b.m))
    short, built = run(N, n, 2), run(n, n, 2)                # a short step on the capacity's buffers vs a step built for n
    assert torch.equal(_bits(short.flat_p), _bits(built.flat_p))
    # state_dict round trip: a new step from a's networks and state continues as a does
    sd = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in a.state_dict().items()}
    nets_c = _nets(G)
    with torch.no_grad():
        for pc, pa in zip([p for m in nets_c for p in m.parameters()], a.params):
            pc.copy_(pa)
    c = FusedTrainStep(400, 400, sb["K"], N, _kwargs(G, nets_c))
    c.load_state_dict(sd)
    a(rays_h, tgt_h)
    c(rays_h, tgt_h)
    assert torch.equal(_bits(a.flat_p), _bits(c.flat_p)) and torch.equal(_bits(a.state), _bits(c.state))
