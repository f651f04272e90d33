"""The short last batch of an epoch, without a GPU: DeviceRayBatcher slices rays_rgb as the reference's train() does
(run_nerf.py:717-726), so when the ray count is not a multiple of N_rand the last batch of each epoch holds the remaining
rays.  FusedTrainStep takes such a batch on the first rows of its buffers (tests/test_gpu_variable_batch.py)."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def nb():
    import __graft_entry__ as ge
    ge.build()
    import nerf_pytorch_b200
    return nerf_pytorch_b200


def test_batcher_yields_the_short_last_batch_of_each_epoch(nb):
    """3 x 1024 + 816 rays at N_rand = 1024: batch sizes 1024, 1024, 1024, 816 per epoch.  Every epoch's batches are its
    rays, each once, in the order of the shuffle that precedes it, and rays_rgb stays the constructor's rays_rgb[perm]."""
    B, n = 1024, 3 * 1024 + 816
    rng = np.random.default_rng(0)
    rays_rgb = rng.random((n, 3, 3), dtype=np.float32)
    images = rng.random((1, 8, 8, 3), dtype=np.float32)
    poses = np.tile(np.eye(4, dtype=np.float32)[:3], (1, 1, 1))
    r0 = torch.from_numpy(rays_rgb)
    torch.manual_seed(5)
    b = nb.DeviceRayBatcher(images, poses, 8, 8, B, rays_rgb=rays_rgb, device="cpu")
    sizes, epoch, order, got = [], [], b.perm.clone(), []
    for _ in range(10):
        rays, target = b.next()
        got.append((rays, target))
        assert rays.shape == (2, target.shape[0], 3) and target.shape[1] == 3
        sizes.append(target.shape[0])
        epoch.append(torch.cat([rays.transpose(0, 1), target[:, None]], 1))
        assert b.perm.dtype == torch.int64 and torch.equal(b.rays_rgb, r0[b.perm])
        if b.i_batch == 0:                                  # an epoch end: its batches are the previous order's rays, once each
            assert torch.equal(torch.cat(epoch), r0[order])
            assert not torch.equal(b.perm, order)
            epoch, order = [], b.perm.clone()
    assert sizes == [1024, 1024, 1024, 816, 1024, 1024, 1024, 816, 1024, 1024]
    # the same batches as the reference's loop with the same seed
    torch.manual_seed(5)
    r, i_batch = r0.clone(), 0
    for rays, target in got:
        batch = r[i_batch:i_batch + B].transpose(0, 1)
        i_batch += B
        if i_batch >= n:
            r = r[torch.randperm(n)]
            i_batch = 0
        assert torch.equal(rays, batch[:2]) and torch.equal(target, batch[2])
