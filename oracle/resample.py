"""Bit-exact float32 restatement of the reference's resampling on CPU torch, plus a float64 variant.

Covers coarse z (run_nerf.py:357-379), sample_pdf (run_nerf_helpers.py:196-239), the merge
sort(cat[z, z_samples]) (run_nerf.py:396) and z_std = std(z_samples, unbiased=False) (:412).

The reference's float32 results depend on how CPU torch rounds three reductions:
  - cumsum accumulates in float64 and rounds every prefix to float32;
  - sum(-1) over a contiguous row of n entries runs in float32 in a fixed order (`torch_sum`);
  - std accumulates in float64 and rounds the result to float32.
tests/test_resample_cpu.py pins these rules to the installed torch.
"""
import numpy as np

VEC = 8          # lanes of the vectorised inner sum (Vectorized<float> of the dispatched kernel)
ILP = 4          # independent accumulators of row_sum
LEVELS = 4       # levels of multi_row_sum's cascade


def _ceil_log2(x):
    return 1 if x <= 2 else int(x - 1).bit_length()


def _multi_row_sum(x):
    """x [N, size, ILP, L] -> [N, ILP, L]: ILP interleaved running sums with a LEVELS-level cascade.
    Every 2^p rows the level-0 sums move up one level; level j moves up every 2^(p*(j+1)) rows."""
    size = x.shape[1]
    p = max(4, _ceil_log2(size) // LEVELS)
    step, mask = 1 << p, (1 << p) - 1
    acc = [np.zeros((x.shape[0],) + x.shape[2:], np.float32) for _ in range(LEVELS)]
    i = 0
    while i + step <= size:
        for _ in range(step):
            acc[0] = acc[0] + x[:, i]
            i += 1
        for j in range(1, LEVELS):
            acc[j] = acc[j] + acc[j - 1]
            acc[j - 1] = np.zeros_like(acc[j - 1])
            if i & (mask << (j * p)):
                break
    while i < size:
        acc[0] = acc[0] + x[:, i]
        i += 1
    for j in range(1, LEVELS):
        acc[0] = acc[0] + acc[j]
    return acc[0]


def _row_sum(x):
    """x [N, size, L] -> [N, L]: ILP accumulators over element k mod ILP, the leftover into the first,
    then the first += the others in order."""
    n_ilp = x.shape[1] // ILP
    part = _multi_row_sum(x[:, :n_ilp * ILP].reshape(x.shape[0], n_ilp, ILP, x.shape[2]))
    p0 = part[:, 0]
    for i in range(n_ilp * ILP, x.shape[1]):
        p0 = p0 + x[:, i]
    for k in range(1, ILP):
        p0 = p0 + part[:, k]
    return p0


def torch_sum(x):
    """float32 x [N, n] -> float32 [N], rounded like CPU torch's x.sum(-1) on a contiguous row.
    n < VEC: scalar row sum.  n >= VEC: row sum over lane-wise VEC-wide vectors, then a scalar total
    that starts at 0, adds the tail x[VEC*V:] in order, then the VEC lanes in order."""
    x = np.ascontiguousarray(x, np.float32)
    N, n = x.shape
    if n < VEC:
        return _row_sum(x[:, :, None])[:, 0]
    V = n // VEC
    lanes = _row_sum(x[:, :V * VEC].reshape(N, V, VEC))
    total = np.zeros(N, np.float32)
    for k in range(V * VEC, n):
        total = total + x[:, k]
    for k in range(VEC):
        total = total + lanes[:, k]
    return total


def torch_cumsum(x):
    """float32 [.., n] -> float32: float64 running sum, each prefix rounded to float32."""
    return np.cumsum(np.asarray(x, np.float64), -1).astype(np.float32)


def torch_linspace(n):
    """torch.linspace(0, 1, n) as CPU torch rounds it (the reference's t_vals and det u)."""
    import torch
    return torch.linspace(0.0, 1.0, steps=n).numpy()


def pytest_linspace(n):
    """The reference's pytest det u: np.linspace(0, 1, n) (float64) through torch.Tensor."""
    return np.linspace(0.0, 1.0, n).astype(np.float32)


def coarse_z(near, far, N_samples, lindisp=False, t_rand=None, dtype=np.float32):
    """near, far [N,1] -> z_vals [N,N_samples] (run_nerf.py:357-379); t_rand [N,N_samples] or None (perturb = 0)."""
    dt = np.dtype(dtype).type
    near, far = np.asarray(near, dtype), np.asarray(far, dtype)
    t = torch_linspace(N_samples).astype(dtype)                                   # :357
    if not lindisp:
        z = near * (dt(1) - t) + far * t                                          # :359
    else:
        z = dt(1) / (dt(1) / near * (dt(1) - t) + dt(1) / far * t)                # :361
    z = np.broadcast_to(z, (near.shape[0], N_samples)).copy()
    if t_rand is not None:
        mids = dt(0.5) * (z[:, 1:] + z[:, :-1])                                   # :367
        upper = np.concatenate([mids, z[:, -1:]], -1)
        lower = np.concatenate([z[:, :1], mids], -1)
        z = lower + (upper - lower) * np.asarray(t_rand, dtype)                   # :379
    return z


def cdf_of(weights, dtype=np.float32):
    """weights [N,B-1] -> cdf [N,B] (run_nerf_helpers.py:198-201).  float32: torch's rounding;
    float64: plain float64 arithmetic."""
    w = np.asarray(weights, dtype) + np.dtype(dtype).type(1e-5)                  # :198
    if dtype == np.float32:
        pdf = w / torch_sum(w)[:, None]                                           # :199
        cdf = torch_cumsum(pdf)                                                   # :200
    else:
        cdf = np.cumsum(w / np.sum(w, -1, keepdims=True), -1)
    return np.concatenate([np.zeros_like(cdf[:, :1]), cdf], -1)                  # :201


def det_u(N_samples, pytest=False):
    return pytest_linspace(N_samples) if pytest else torch_linspace(N_samples)


def sample_pdf(bins, weights, N_samples, det=False, u=None, pytest=False, dtype=np.float32):
    """bins [N,B], weights [N,B-1] -> samples [N,N_samples] (run_nerf_helpers.py:196-239).
    `u` [N,N_samples] replaces the random draw; det without `u` uses the reference's linspace
    (numpy's on its pytest path, torch's otherwise)."""
    dt = np.dtype(dtype).type
    bins = np.asarray(bins, dtype)
    cdf = cdf_of(weights, dtype)
    N, B = cdf.shape
    if u is None:
        assert det, "random u must be injected"
        u = det_u(N_samples, pytest)
    u = np.ascontiguousarray(np.broadcast_to(np.asarray(u, np.float32).astype(dtype), (N, N_samples)))
    inds = np.stack([np.searchsorted(cdf[i], u[i], side="right") for i in range(N)])   # :223
    below = np.maximum(0, inds - 1)                                               # :224
    above = np.minimum(B - 1, inds)                                               # :225
    c0, c1 = np.take_along_axis(cdf, below, -1), np.take_along_axis(cdf, above, -1)
    b0, b1 = np.take_along_axis(bins, below, -1), np.take_along_axis(bins, above, -1)
    denom = c1 - c0                                                               # :234
    denom = np.where(denom < dt(1e-5), np.ones_like(denom), denom)                # :235
    t = (u - c0) / denom                                                          # :236
    return b0 + t * (b1 - b0)                                                     # :237


def merge(z_vals, z_samples):
    """sort(cat[z_vals, z_samples], -1) (run_nerf.py:396)."""
    return np.sort(np.concatenate([z_vals, z_samples], -1), -1)


def z_std(z_samples):
    """std(z_samples, -1, unbiased=False) (run_nerf.py:412): float64, rounded to the input's type."""
    s = np.asarray(z_samples)
    return np.std(s.astype(np.float64), -1).astype(s.dtype)


def fine_z(z_vals, weights, N_importance, det=False, u=None, pytest=False, dtype=np.float32):
    """Hierarchical resampling of render_rays (run_nerf.py:392-396, :412):
    z_vals, weights [N,S] -> (z_fine [N,S+N_importance], z_samples [N,N_importance], z_std [N])."""
    dt = np.dtype(dtype).type
    z = np.asarray(z_vals, dtype)
    mid = dt(0.5) * (z[:, 1:] + z[:, :-1])                                        # :392
    s = sample_pdf(mid, np.asarray(weights, dtype)[:, 1:-1], N_importance, det, u, pytest, dtype)
    return merge(z, s), s, z_std(s)
