"""Generate tests/golden/resample.npz by running the UNMODIFIED reference on CPU  --  build container only.

    python oracle/gen_resample_golden.py      # needs the reference checkout (oracle/ref_import.py); writes tests/golden/

Two kinds of cases, all float32:

  p{i}_*  sample_pdf (run_nerf_helpers.py:196-239) on bins [R,B] / weights [R,B-1], one row per weight profile (PROFILES):
          p{i}_meta = [B, n, u kind] with kinds  0 torch.linspace (det), 1 np.linspace (det, the pytest path),
          2 random u, 3 u on cdf knots (each row's own cdf entries, duplicated, plus 0 and 1, in random order).
          p{i}_u is the [n] row (kinds 0, 1) or [R,n]; p{i}_out the reference's samples.
  f{i}_*  render_rays' resampling (run_nerf.py:357-412) through the reference's own render_rays, with a stub network
          query that returns a stored coarse raw and records the fine z: rays start at 0 along +z, so
          pts[..., 2] == z exactly.  f{i}_meta = [S, N_importance, lindisp, perturb]; inputs near/far [N],
          t_rand [N,S] and u [N,Ni] (perturb only); outputs z_coarse, w_coarse, z_fine, z_std.

There is no S = 2 case: with N_importance > 0 the reference fails there (weights[..., 1:-1] is empty, so its cdf has no
entry and torch.gather raises), and nerf_b200_fine_z refuses S < 3 likewise.

torch.rand is the reference's only random draw on these paths; it is replaced for the call by a function that returns
the injected arrays in draw order (t_rand, then u).
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
U_TORCH, U_PYTEST, U_RAND, U_KNOTS = 0, 1, 2, 3
PROFILES = ("random", "cubed", "zero", "onehot_first", "onehot_mid", "onehot_last", "peak_then_zeros", "leading_zeros",
            "tiny", "large", "equal")
SPDF = [(2, 128, U_TORCH), (3, 31, U_RAND), (5, 2, U_KNOTS), (8, 32, U_PYTEST), (9, 1, U_TORCH), (9, 128, U_KNOTS),
        (33, 33, U_RAND), (63, 128, U_KNOTS), (63, 128, U_RAND), (63, 128, U_PYTEST), (64, 1000, U_TORCH),
        (65, 128, U_PYTEST), (129, 31, U_KNOTS), (257, 33, U_TORCH), (513, 128, U_RAND), (513, 32, U_KNOTS)]
# S, N_importance, lindisp, perturb, N rays, t_rand pattern
FINE = [(64, 128, 0, 0, 24, None), (64, 128, 0, 1, 24, "edges"), (8, 16, 0, 1, 4, "ties"),
        (33, 31, 1, 1, 8, "edges"), (3, 1, 0, 0, 5, None)]


def weight_rows(rng, n):
    """[len(PROFILES), n] non-negative weights, one row per profile."""
    rows = []
    for p in PROFILES:
        w = np.zeros(n, np.float32)
        if p == "random":
            w = rng.random(n, dtype=np.float32)
        elif p == "cubed":
            w = rng.random(n, dtype=np.float32) ** 3
        elif p in ("onehot_first", "onehot_mid", "onehot_last") and n > 0:
            w[{"onehot_first": 0, "onehot_mid": n // 2, "onehot_last": n - 1}[p]] = 1.0
        elif p == "peak_then_zeros" and n > 0:        # an opaque ray: everything behind the surface is exactly 0
            k = n // 3
            w[:k] = 0.01 * rng.random(k, dtype=np.float32)
            w[k] = 0.9
        elif p == "leading_zeros":
            w[n // 2:] = rng.random(n - n // 2, dtype=np.float32)
        elif p == "tiny":
            w[:] = 1e-30
        elif p == "large":
            w = (1e3 * rng.random(n, dtype=np.float32)).astype(np.float32)
        elif p == "equal":
            w[:] = 0.5
        rows.append(w.astype(np.float32))
    return np.stack(rows)


def bin_rows(rng, R, B):
    """[R, B] strictly ascending bins in [2, 6], like z midpoints."""
    g = np.cumsum(0.2 + rng.random((R, B)), -1)
    return (2.0 + 4.0 * (g - g[:, :1]) / np.maximum(g[:, -1:] - g[:, :1], 1e-9)).astype(np.float32)


class InjectRand:
    """torch.rand -> the given arrays, in call order."""
    def __init__(self, *arrays):
        self.arrays = list(arrays)

    def __enter__(self):
        self.saved = torch.rand
        torch.rand = lambda *a, **k: torch.from_numpy(self.arrays.pop(0).copy())
        return self

    def __exit__(self, *exc):
        torch.rand = self.saved
        assert not self.arrays, "unused injected draws"


def knot_u(rng, w, n):
    """[R, n]: each row's cdf entries (as the reference computes them), some duplicated, plus 0 and 1, shuffled."""
    wt = torch.from_numpy(w) + 1e-5
    cdf = torch.cumsum(wt / torch.sum(wt, -1, keepdim=True), -1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1).numpy()
    u = cdf[np.arange(cdf.shape[0])[:, None], rng.integers(0, cdf.shape[1], (cdf.shape[0], n))]
    if n >= 2:
        u[:, 0], u[:, 1] = 0.0, 1.0
    if n >= 4:
        u[:, 3] = u[:, 2]
    for r in range(u.shape[0]):
        rng.shuffle(u[r])
    return np.ascontiguousarray(u, np.float32)


def run_spdf(rh, fx, i, B, n, kind, rng):
    w = weight_rows(rng, B - 1)
    bins = bin_rows(rng, w.shape[0], B)
    tb, tw = torch.from_numpy(bins), torch.from_numpy(w)
    if kind == U_TORCH:
        out, u = rh.sample_pdf(tb, tw, n, det=True), torch.linspace(0., 1., steps=n).numpy()
    elif kind == U_PYTEST:
        out, u = rh.sample_pdf(tb, tw, n, det=True, pytest=True), np.linspace(0., 1., n).astype(np.float32)
    else:
        u = rng.random((w.shape[0], n), dtype=np.float32) if kind == U_RAND else knot_u(rng, w, n)
        with InjectRand(u):
            out = rh.sample_pdf(tb, tw, n, det=False)
    p = f"p{i}_"
    fx[p + "meta"] = np.array([B, n, kind], np.int32)
    fx[p + "bins"], fx[p + "w"], fx[p + "u"], fx[p + "out"] = bins, w, np.asarray(u, np.float32), out.numpy()


def run_fine(rn, fx, i, S, Ni, lindisp, perturb, N, pattern, rng):
    near = (1.0 + 2.0 * rng.random(N, dtype=np.float32)).astype(np.float32)
    far = (near + 2.0 + 4.0 * rng.random(N, dtype=np.float32)).astype(np.float32)
    rays = np.zeros((N, 8), np.float32)
    rays[:, 5], rays[:, 6], rays[:, 7] = 1.0, near, far
    raw = rng.standard_normal((N, S, 4), dtype=np.float32)
    raw[::3, :, 3] = np.abs(raw[::3, :, 3]) * 40.0          # every third ray opaque: its trailing weights are exactly 0
    draws = []
    if perturb:
        t_rand = rng.random((N, S), dtype=np.float32)
        if pattern == "edges":
            t_rand[:, 0], t_rand[:, -1], t_rand[1::2, 1] = 0.0, 1.0, 1.0
        elif pattern == "ties":                             # 1 then 0: z[s] = upper_s = mid = lower_{s+1} = z[s+1]
            t_rand[:, 0::2], t_rand[:, 1::2] = 1.0, 0.0
        u = rng.random((N, Ni), dtype=np.float32)
        draws = [t_rand, u]
    seen = []

    def query(pts, viewdirs, fn):
        seen.append(pts[..., 2].clone())
        return torch.from_numpy(raw) if len(seen) == 1 else torch.zeros(pts.shape[:-1] + (4,))

    with InjectRand(*draws):
        ret = rn.render_rays(torch.from_numpy(rays), None, query, S, lindisp=bool(lindisp), perturb=float(perturb),
                             N_importance=Ni, network_fine=None)
    z_coarse, z_fine = seen[0], seen[1]
    w_coarse = rn.raw2outputs(torch.from_numpy(raw), z_coarse, torch.from_numpy(rays[:, 3:6]))[3]
    p = f"f{i}_"
    fx[p + "meta"] = np.array([S, Ni, lindisp, perturb], np.int32)
    fx[p + "near"], fx[p + "far"] = near, far
    if perturb:
        fx[p + "t_rand"], fx[p + "u"] = draws
    fx[p + "z_coarse"], fx[p + "w_coarse"] = z_coarse.numpy(), w_coarse.numpy()
    fx[p + "z_fine"], fx[p + "z_std"] = z_fine.numpy(), ret["z_std"].numpy()


def main():
    assert ref_import.available(), "reference not found (this script only runs where the reference checkout exists)"
    t0 = time.time()
    torch.set_num_threads(8)
    rn, rh = ref_import.load()
    rng = np.random.default_rng(20261017)
    fx = {}
    for i, (B, n, kind) in enumerate(SPDF):
        run_spdf(rh, fx, i, B, n, kind, rng)
    for i, c in enumerate(FINE):
        run_fine(rn, fx, i, *c, rng)
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "resample.npz"), **fx)
    print("wrote resample", len(fx), "arrays in", round(time.time() - t0, 1), "s")


if __name__ == "__main__":
    main()
