"""The torch decoder of the tile records (tests/tc_records.py gather_image_t / gather_mask_t, which the full-plan GPU tests run
on the device) against the numpy decoder, on random record bytes and tile plans with ragged CTAs and empty tiles."""
import numpy as np
import pytest
import torch

import tc_records as R

D = 2


# (N, S, SMs): what each plan holds
PLANS = [(10, 100, 4),     # last CTA one ray of three; a CTA's second super-tile ends inside its first tile (empty second tile)
         (12, 128, 4),     # rays_per_cta * S = 384 = 128 mod 256: the last super-tile of every CTA has an empty second tile
         (7, 128, 4),      # last CTA one ray: half of the record stride, its second tile empty
         (9, 40, 2),       # S not a multiple of 8, rays straddle tiles
         (3, 300, 8)]      # grid clamped to N, a ray over two super-tiles


def _plan(N, S, sms):
    layout, _, _ = R.restate_layout(N, S, D, 27, sms)
    return R.Plan(None, N, S, None, layout=layout)


@pytest.mark.parametrize("N,S,sms", PLANS)
def test_torch_decoder_is_the_numpy_decoder(N, S, sms):
    plan = _plan(N, S, sms)
    assert not R.plan_row_keep(plan).all(), "the plan must leave rows of its valid tiles unused"
    rng = np.random.default_rng(N * 1000 + S)
    act = rng.integers(0, 256, plan.n_tiles * plan.rec_act, dtype=np.uint8)
    mask = rng.integers(0, 256, plan.n_tiles * plan.rec_mask, dtype=np.uint8)
    act_t, mask_t = torch.from_numpy(act), torch.from_numpy(mask)
    for off, ncol in [(0, 64)] + [(R.rec_act_h(l), 256) for l in range(D)] + [(R.rec_act_h(D), 128)]:
        ref = R.gather_image(act, plan, plan.rec_act, off, ncol)
        got = R.gather_image_t(act_t, plan, plan.rec_act, off, ncol)
        assert got.dtype == torch.float16 and got.shape == (N * S, ncol)
        # random bytes hold NaNs: compare the fp16 bit patterns (float32 <- fp16 is exact and keeps them)
        assert np.array_equal(ref.astype(np.float16).view(np.uint16), got.numpy().view(np.uint16)), (off, ncol)
    for l in range(D):
        assert np.array_equal(R.gather_mask(mask, plan, l, D), R.gather_mask_t(mask_t, plan, l, D).numpy()), l
    assert np.array_equal(R.gather_mask(mask, plan, 0, D, hv=True), R.gather_mask_t(mask_t, plan, 0, D, hv=True).numpy())


def test_plans_cover_ragged_and_empty_tiles():
    """the plans above hold what they are listed for"""
    p = _plan(10, 100, 4)
    assert (p.grid, p.rays_per_cta, p.nst) == (4, 3, 2) and p.cta_nst(3) == 1
    p = _plan(12, 128, 4)
    assert p.rays_per_cta * 128 % 256 == 128 and (p.rows_of_tile(3) < 0).all()
    p = _plan(7, 128, 4)
    assert p.N - (p.grid - 1) * p.rays_per_cta == 1 and (p.rows_of_tile(2 * (p.grid - 1) + 1) < 0).all()
