"""Resuming training, without a GPU: trainer.adam_moments (the mapping FusedTrainStep.load_optimizer uses) finds each
parameter's Adam state by identity and refuses what the flat Adam cannot continue from; DeviceRayBatcher keeps the order of
its rays as a permutation and continues from its state_dict to the same batches."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def nb():
    import __graft_entry__ as ge
    ge.build()
    import nerf_pytorch_b200
    return nerf_pytorch_b200


@pytest.fixture(scope="module")
def T(nb):
    from nerf_pytorch_b200 import trainer
    return trainer


def _nets(nb, views=True):
    torch.manual_seed(0)
    return [nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27 if views else 0, output_ch=5, skips=[4], use_viewdirs=views)
            for _ in range(2)]


def _named(nets):
    """(name, parameter) in FusedTrainStep's flat order"""
    return [(f"{tag}.{k}", p) for tag, n in zip(("network_fn", "network_fine"), nets) for k, p in n.named_parameters()]


def _trained_adam(params, steps=3, groups=None):
    """torch.optim.Adam after `steps` steps of a loss whose gradient differs per element"""
    opt = torch.optim.Adam(groups if groups is not None else params, lr=5e-4, betas=(0.9, 0.999))
    g = torch.Generator().manual_seed(1)
    w = [torch.randn(p.shape, generator=g) for p in params]
    for _ in range(steps):
        opt.zero_grad()
        sum(((p * c) ** 2).sum() + (p * c).sum() for p, c in zip(params, w)).backward()
        opt.step()
    return opt


@pytest.mark.parametrize("views", [True, False])
def test_moments_map_to_flat_offsets_by_identity(nb, T, views):
    """The optimizer lists the parameters in another order and in two groups: each moment still lands at its parameter's offset."""
    nets = _nets(nb, views)
    named = _named(nets)
    params = [p for _, p in named]
    shuffled = params[::-1]
    opt = _trained_adam(params, groups=[{"params": shuffled[:17]}, {"params": shuffled[17:]}])
    step, moments = T.adam_moments(named, opt, (0.9, 0.999), 1e-8)
    assert step == 3 and len(moments) == len(params)
    m_flat, v_flat = torch.zeros(sum(p.numel() for p in params)), torch.zeros(sum(p.numel() for p in params))
    for off, m, v in moments:
        m_flat[off:off + m.numel()] = m.reshape(-1)
        v_flat[off:off + v.numel()] = v.reshape(-1)
    off = 0
    for p in params:
        assert torch.equal(m_flat[off:off + p.numel()], opt.state[p]["exp_avg"].reshape(-1))
        assert torch.equal(v_flat[off:off + p.numel()], opt.state[p]["exp_avg_sq"].reshape(-1))
        off += p.numel()
    assert off == m_flat.numel() and bool((v_flat > 0).all())


def test_shared_fine_net_is_counted_once(nb, T):
    net = _nets(nb)[0]
    named = [(f"network_fn.{k}", p) for k, p in net.named_parameters()]
    opt = _trained_adam([p for _, p in named])
    step, moments = T.adam_moments(named, opt, (0.9, 0.999), 1e-8)
    assert step == 3 and [o for o, _, _ in moments] == list(np.cumsum([0] + [p.numel() for _, p in named])[:-1])


def test_step_as_int_or_tensor(nb, T):
    """torch 1.11 (which the reference pins) keeps Adam's step as an int, current torch as a tensor"""
    nets = _nets(nb)
    named = _named(nets)
    opt = _trained_adam([p for _, p in named], steps=2)
    assert torch.is_tensor(opt.state[named[0][1]]["step"])
    as_tensor = T.adam_moments(named, opt, (0.9, 0.999), 1e-8)
    for _, p in named:
        opt.state[p]["step"] = 2
    as_int = T.adam_moments(named, opt, (0.9, 0.999), 1e-8)
    assert as_tensor[0] == as_int[0] == 2
    assert all(a[0] == b[0] and a[1] is b[1] for a, b in zip(as_tensor[1], as_int[1]))


def test_empty_state_is_none(nb, T):
    named = _named(_nets(nb))
    opt = torch.optim.Adam([p for _, p in named], lr=5e-4)
    assert T.adam_moments(named, opt, (0.9, 0.999), 1e-8) is None


def _refusal(nb, T, spoil):
    named = _named(_nets(nb))
    params = [p for _, p in named]
    opt = _trained_adam(params, steps=2)
    betas, eps = spoil(opt, params) or ((0.9, 0.999), 1e-8)
    with pytest.raises(RuntimeError) as e:
        T.adam_moments(named, opt, betas, eps)
    return str(e.value)


def test_refuses_a_parameter_missing_from_the_optimizer(nb, T):
    def spoil(opt, params):
        opt.param_groups[0]["params"] = [q for q in opt.param_groups[0]["params"] if q is not params[5]]
    assert "network_fn.pts_linears.2.bias is not in the optimizer" in _refusal(nb, T, spoil)


def test_refuses_a_moment_of_another_shape(nb, T):
    def spoil(opt, params):
        opt.state[params[30]]["exp_avg_sq"] = opt.state[params[30]]["exp_avg_sq"].reshape(-1)[:10]
    msg = _refusal(nb, T, spoil)
    assert "exp_avg_sq of network_fine." in msg and "shape (10,)" in msg


def test_refuses_moments_for_some_parameters_only(nb, T):
    def spoil(opt, params):
        del opt.state[params[7]]
    msg = _refusal(nb, T, spoil)
    assert "for 47 of 48 parameters" in msg and "network_fn.pts_linears.3.bias" in msg


def test_refuses_unequal_step_counts(nb, T):
    def spoil(opt, params):
        opt.state[params[40]]["step"] = torch.tensor(5.0)
    msg = _refusal(nb, T, spoil)
    assert "step counts differ" in msg and "5 (network_fine." in msg


@pytest.mark.parametrize("what", ["beta1", "beta2", "eps", "step_betas", "step_eps"])
def test_refuses_other_betas_or_eps(nb, T, what):
    def spoil(opt, params):
        g = opt.param_groups[0]
        if what == "beta1":
            g["betas"] = (0.8, 0.999)
        elif what == "beta2":
            g["betas"] = (0.9, 0.99)
        elif what == "eps":
            g["eps"] = 1e-7
        elif what == "step_betas":
            return (0.9, 0.99), 1e-8
        else:
            return (0.9, 0.999), 1e-6
    assert "differ from the step's own" in _refusal(nb, T, spoil)


def test_refuses_weight_decay(nb, T):
    def spoil(opt, params):
        opt.param_groups[0]["weight_decay"] = 1e-4
    assert "weight_decay" in _refusal(nb, T, spoil)


def test_refuses_a_step_count_that_is_not_whole(nb, T):
    def spoil(opt, params):
        for p in params:
            opt.state[p]["step"] = 2.5
    assert "not a whole number" in _refusal(nb, T, spoil)


# ---- DeviceRayBatcher ------------------------------------------------------------------------------------------------------

def _data(n_img=6, H=8, W=8):
    rng = np.random.default_rng(0)
    images = rng.random((n_img, H, W, 3), dtype=np.float32)
    poses = np.tile(np.eye(4, dtype=np.float32)[:3], (n_img, 1, 1))
    poses[:, :, 3] = rng.random((n_img, 3), dtype=np.float32)
    rays_rgb = rng.random((n_img * H * W, 3, 3), dtype=np.float32)
    return images, poses, H, W, rays_rgb


def _batches(b, n):
    return [tuple(x.clone() for x in b.next()) for _ in range(n)]


def test_batcher_keeps_the_order_as_a_permutation_and_next_is_unchanged(nb):
    """rays_rgb == the constructor's rays_rgb[perm] across epoch ends, and the batches are those of the shuffle-the-rays loop of
    train() (run_nerf.py:717-726) with the same seed"""
    images, poses, H, W, rays_rgb = _data()
    B, n = 96, rays_rgb.shape[0]                        # 384 rays: an epoch end every 4 steps
    r0 = torch.from_numpy(rays_rgb)
    torch.manual_seed(5)
    b = nb.DeviceRayBatcher(images, poses, H, W, B, rays_rgb=rays_rgb, device="cpu")
    got = []
    for _ in range(11):
        got.append(b.next())
        assert b.perm.dtype == torch.int64 and torch.equal(b.rays_rgb, r0[b.perm])
    assert not torch.equal(b.perm, torch.arange(n))
    torch.manual_seed(5)
    r, i_batch = r0.clone(), 0
    for rays, target in got:
        batch = r[i_batch:i_batch + B].transpose(0, 1)
        i_batch += B
        if i_batch >= n:
            r = r[torch.randperm(n)]
            i_batch = 0
        assert torch.equal(rays, batch[:2]) and torch.equal(target, batch[2])


@pytest.mark.parametrize("mode", ["rays", "pixels"])
def test_batcher_continues_from_its_state_dict(nb, mode):
    """k batches, state_dict, then the same batches from a new batcher (or one that has moved on) loaded with that state.  On
    the CPU every draw of next() is the host generator's, which the state holds."""
    images, poses, H, W, rays_rgb = _data()
    kw = dict(rays_rgb=rays_rgb) if mode == "rays" else dict(i_train=[0, 2, 3, 5], precrop_iters=6, precrop_frac=0.5)
    torch.manual_seed(3)
    a = nb.DeviceRayBatcher(images, poses, H, W, 96, device="cpu", **kw)
    _batches(a, 5)                                      # (rays: across an epoch end; pixels: inside the crop)
    sd = a.state_dict()
    assert sd["step"] == 5 and (sd["perm"] is None) == (mode == "pixels")
    want = _batches(a, 7)                               # (rays: across the next epoch end; pixels: the crop ends)
    for fresh in (True, False):
        torch.manual_seed(99)
        b = nb.DeviceRayBatcher(images, poses, H, W, 96, device="cpu", **kw)
        if not fresh:
            _batches(b, 6)
        b.load_state_dict(sd)
        got = _batches(b, 7)
        for x, y in zip(want, got):
            assert all(torch.equal(u, v) for u, v in zip(x, y))


def test_batcher_refuses_a_foreign_state(nb):
    images, poses, H, W, rays_rgb = _data()
    a = nb.DeviceRayBatcher(images, poses, H, W, 96, rays_rgb=rays_rgb, device="cpu")
    p = nb.DeviceRayBatcher(images, poses, H, W, 96, device="cpu")
    with pytest.raises(RuntimeError, match="other batching mode"):
        p.load_state_dict(a.state_dict())
    with pytest.raises(RuntimeError, match="other batching mode"):
        a.load_state_dict(p.state_dict())
    sd = a.state_dict()
    for bad in (torch.zeros(rays_rgb.shape[0], dtype=torch.int64), torch.arange(rays_rgb.shape[0] - 1), torch.arange(rays_rgb.shape[0]).int()):
        with pytest.raises(RuntimeError, match="not an int64 permutation"):
            a.load_state_dict(dict(sd, perm=bad))
    with pytest.raises(RuntimeError, match="outside"):
        a.load_state_dict(dict(sd, i_batch=rays_rgb.shape[0]))
