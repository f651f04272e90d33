"""oracle/resample.py, the float32 restatement of the reference's resampling, equals the reference bit for bit:
against the recorded fixtures (units.npz, trained_lego_1024.npz, resample.npz from oracle/gen_resample_golden.py) and
against the same torch ops evaluated live on CPU, which pins its sum / cumsum / std rounding rules to the installed torch.
CPU only."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import nerf_oracle as O
from oracle import resample as R


def eq(a, b):
    """bit-equal float32 arrays (NaN never expected here)"""
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def spdf_cases():
    fx = load_golden("resample")
    return [(i, fx) for i in range(len([k for k in fx if k.startswith("p") and k.endswith("_meta")]))]


def fine_cases():
    fx = load_golden("resample")
    return [(i, fx) for i in range(len([k for k in fx if k.startswith("f") and k.endswith("_meta")]))]


def golden_spdf(fx, i):
    B, n, kind = (int(v) for v in fx[f"p{i}_meta"])
    u = fx[f"p{i}_u"]
    return fx[f"p{i}_bins"], fx[f"p{i}_w"], n, kind, (np.broadcast_to(u, (fx[f"p{i}_w"].shape[0], n)) if u.ndim == 1 else u)


# ---- the recorded reference ----------------------------------------------------------------------------------------

def test_units_sample_pdf_bit_exact():
    fx = load_golden("units")
    assert eq(R.sample_pdf(fx["spdf_bins"], fx["spdf_w"], 128, det=True), fx["spdf_det"])
    assert eq(R.sample_pdf(fx["spdf_bins"], fx["spdf_w"], 128, u=fx["spdf_u"]), fx["spdf_rand"])


def test_trained_lego_resampling_bit_exact():
    """The reference's own coarse z and weights of 1024 trained-net rays -> its z_fine and z_std."""
    fx = load_golden("trained_lego_1024")
    N = fx["z_coarse"].shape[0]
    assert eq(R.coarse_z(np.full((N, 1), 2.0, np.float32), np.full((N, 1), 6.0, np.float32), 64), fx["z_coarse"])
    z_fine, _, z_std = R.fine_z(fx["z_coarse"], fx["w_coarse"], 128, det=True)
    assert eq(z_fine, fx["z_fine"]) and eq(z_std, fx["z_std"])


def test_resample_golden_covers_the_matrix():
    fx = load_golden("resample")
    metas = [fx[f"p{i}_meta"] for i, _ in spdf_cases()]
    assert {int(m[0]) for m in metas} == {2, 3, 5, 8, 9, 33, 63, 64, 65, 129, 257, 513}
    assert {int(m[1]) for m in metas} == {1, 2, 31, 32, 33, 128, 1000}
    assert {int(m[2]) for m in metas} == {0, 1, 2, 3}
    fm = [fx[f"f{i}_meta"] for i, _ in fine_cases()]
    assert any(m[2] for m in fm) and any(m[3] for m in fm) and any(not m[3] for m in fm)
    ties = [i for i, _ in fine_cases() if (np.diff(fx[f"f{i}_z_coarse"], axis=-1) == 0).any()]
    assert ties, "one case must merge equal coarse neighbours"


@pytest.mark.parametrize("i,fx", spdf_cases(), ids=lambda v: str(v) if isinstance(v, int) else "")
def test_sample_pdf_golden_bit_exact(i, fx):
    bins, w, n, kind, u = golden_spdf(fx, i)
    assert eq(R.sample_pdf(bins, w, n, u=u), fx[f"p{i}_out"])
    if kind in (0, 1):                    # the det paths draw their own linspace
        assert eq(R.sample_pdf(bins, w, n, det=True, pytest=kind == 1), fx[f"p{i}_out"])
        assert eq(O.sample_pdf(bins, w, n, det=True, pytest=kind == 1), fx[f"p{i}_out"])
    else:
        assert eq(O.sample_pdf(bins, w, n, u=u), fx[f"p{i}_out"])


@pytest.mark.parametrize("i,fx", fine_cases(), ids=lambda v: str(v) if isinstance(v, int) else "")
def test_fine_z_golden_bit_exact(i, fx):
    p = f"f{i}_"
    S, Ni, lindisp, perturb = (int(v) for v in fx[p + "meta"])
    z = R.coarse_z(fx[p + "near"][:, None], fx[p + "far"][:, None], S, bool(lindisp), fx.get(p + "t_rand"))
    assert eq(z, fx[p + "z_coarse"])
    z_fine, s, z_std = R.fine_z(z, fx[p + "w_coarse"], Ni, det=not perturb, u=fx.get(p + "u"))
    assert eq(z_fine, fx[p + "z_fine"]) and eq(z_std, fx[p + "z_std"])


# ---- the rules against live CPU torch --------------------------------------------------------------------------

SUM_SIZES = list(range(0, 70)) + [126, 127, 128, 255, 256, 257, 511, 512, 513, 543, 544, 1023, 1024, 2047, 2048,
                                  4093, 4095]


@pytest.mark.parametrize("n", SUM_SIZES)
def test_sum_order_matches_torch(n):
    """torch's float32 sum over the whole range sample_pdf (B - 1 <= 2047) and fine_z (S - 2 <= 4093) reach."""
    rng = np.random.default_rng(n)
    x = np.concatenate([rng.random((64, n), dtype=np.float32) ** 3, 1e3 * rng.random((64, n), dtype=np.float32),
                        rng.random((64, n), dtype=np.float32) * (rng.random((64, n)) < 0.1)]).astype(np.float32) + np.float32(1e-5)
    assert eq(R.torch_sum(x), torch.from_numpy(x).sum(-1).numpy())


@pytest.mark.parametrize("n", [1, 2, 31, 62, 127, 512, 2047, 4093])
def test_cumsum_and_std_match_torch(n):
    rng = np.random.default_rng(100 + n)
    x = (rng.random((128, n), dtype=np.float32) ** 2 / np.float32(n)).astype(np.float32)
    assert eq(R.torch_cumsum(x), torch.cumsum(torch.from_numpy(x), -1).numpy())
    z = (2 + 4 * rng.random((128, n), dtype=np.float32)).astype(np.float32)
    assert eq(R.z_std(z), torch.std(torch.from_numpy(z), dim=-1, unbiased=False).numpy())


def torch_sample_pdf(bins, weights, u):
    """run_nerf_helpers.py:198-237 in torch with an injected u (the ops of the reference, evaluated live)."""
    bins, weights, u = (torch.from_numpy(np.ascontiguousarray(a)) for a in (bins, weights, u))
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cat([torch.zeros_like(pdf[..., :1]), torch.cumsum(pdf, -1)], -1)
    inds = torch.searchsorted(cdf, u.contiguous(), right=True)
    below = torch.clamp(inds - 1, min=0)
    above = torch.clamp(inds, max=cdf.shape[-1] - 1)
    c0, c1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    b0, b1 = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = c1 - c0
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    return (b0 + (u - c0) / denom * (b1 - b0)).numpy()


@pytest.mark.parametrize("B", [2, 4, 9, 40, 63, 200, 600, 1100, 2048])
def test_sample_pdf_matches_torch(B):
    rng = np.random.default_rng(B)
    R_ = 48
    w = rng.random((R_, B - 1), dtype=np.float32) ** 4
    w[::4, (B - 1) // 2:] = 0.0                            # opaque rows: exact zeros behind a peak
    bins = np.sort(2 + 4 * rng.random((R_, B), dtype=np.float32), -1).astype(np.float32)
    u = rng.random((R_, 160), dtype=np.float32)
    u[:, :2] = [0.0, 1.0]
    assert eq(R.sample_pdf(bins, w, 160, u=u), torch_sample_pdf(bins, w, u))


def test_linspaces():
    """torch.linspace and the pytest path's np.linspace differ; the restatement keeps both."""
    t = R.torch_linspace(128)
    assert eq(t, torch.linspace(0., 1., 128).numpy())
    assert not eq(t, R.pytest_linspace(128))


def test_float64_variant_is_close():
    fx = load_golden("trained_lego_1024")
    z32, _, s32 = R.fine_z(fx["z_coarse"], fx["w_coarse"], 128, det=True)
    z64, _, s64 = R.fine_z(fx["z_coarse"], fx["w_coarse"], 128, det=True, dtype=np.float64)
    assert z64.dtype == np.float64 and s64.dtype == np.float64
    assert np.linalg.norm(z32 - z64) / np.linalg.norm(z64) < 1e-3


# ---- the fixtures tell the rules apart -----------------------------------------------------------------------------

def _warp_total(x):
    """a warp's sum: lane-strided float32 partial sums, then the xor butterfly (common.cuh warp_sum)"""
    N, n = x.shape
    lanes = np.zeros((N, 32), np.float32)
    for i in range(n):
        lanes[:, i % 32] = lanes[:, i % 32] + x[:, i]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    return lanes[:, 0]


def _variant_sample_pdf(bins, w, u, total=R.torch_sum, cumsum=R.torch_cumsum, side="right"):
    x = np.asarray(w, np.float32) + np.float32(1e-5)
    cdf = cumsum(x / total(x)[:, None])
    cdf = np.concatenate([np.zeros_like(cdf[:, :1]), cdf], -1)
    inds = np.stack([np.searchsorted(cdf[i], u[i], side=side) for i in range(cdf.shape[0])])
    below, above = np.maximum(0, inds - 1), np.minimum(cdf.shape[1] - 1, inds)
    c0, c1 = np.take_along_axis(cdf, below, -1), np.take_along_axis(cdf, above, -1)
    b0, b1 = np.take_along_axis(bins, below, -1), np.take_along_axis(bins, above, -1)
    denom = c1 - c0
    denom = np.where(denom < np.float32(1e-5), np.ones_like(denom), denom)
    return b0 + (u - c0) / denom * (b1 - b0)


@pytest.mark.parametrize("variant", ["float32_cumsum", "warp_total", "searchsorted_left"])
def test_fixtures_reject_other_rounding(variant):
    """A float32 sequential cumsum, a warp-reduction total or searchsorted(right=False) each miss the recorded reference:
    bit-exact tests on these fixtures fail for a kernel with any of them."""
    kw = {"float32_cumsum": dict(cumsum=lambda p: np.cumsum(p, -1, dtype=np.float32)),
          "warp_total": dict(total=_warp_total), "searchsorted_left": dict(side="left")}[variant]
    fx = load_golden("resample")
    missed = []
    for i, _ in spdf_cases():
        bins, w, n, kind, u = golden_spdf(fx, i)
        assert eq(_variant_sample_pdf(bins, w, u), fx[f"p{i}_out"])            # the helper itself is the reference's
        if not eq(_variant_sample_pdf(bins, w, u, **kw), fx[f"p{i}_out"]):
            missed.append(i)
    tl = load_golden("trained_lego_1024")
    z = tl["z_coarse"]
    mid, u = np.float32(0.5) * (z[:, 1:] + z[:, :-1]), np.broadcast_to(R.torch_linspace(128), (z.shape[0], 128))
    trained_moves = not eq(_variant_sample_pdf(mid, tl["w_coarse"][:, 1:-1], u, **kw),
                           _variant_sample_pdf(mid, tl["w_coarse"][:, 1:-1], u))
    assert missed and (trained_moves or variant == "searchsorted_left"), (missed, trained_moves)
