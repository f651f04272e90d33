"""Generate tests/golden/vertex_attrs.npz by running the UNMODIFIED reference on CPU  --  build container only.

    python oracle/gen_vertex_golden.py        # needs the reference checkout (oracle/ref_import.py); writes tests/golden/

The vertex attributes a mesh export needs, the way the reference gives them: the density gradient by ordinary autograd through
its own network_query_fn (run_network), torch.autograd.grad(run_network(pts)[..., 3].sum(), pts), and the colour of the view
head looking along that gradient, sigmoid(run_network(pts, viewdirs = grad / |grad|)[..., :3]).  The nets are

    c, f : the trained coarse and fine nets of trained_weights.npz (view directions)
    nv   : a net without view directions (output_ch 5) with the trained fine net's density (oracle/outgrads.noviews_from_trained)

Points per net: UNIFORM uniform points in [-1.3, 1.3]^3, then the level crossings (sigma = ISO) of the reference's own float32
sigma on a coarse GRID^3 grid over the same cube, one per crossing grid edge, found by linear interpolation in numpy (so the
fixture does not depend on the library's marching cubes), at most NEAR of them.

Stored per net n: `<n>_pts` [P, 3] float32, `<n>_sigma` [P] (the reference in float32), `<n>_grad` [P, 3] (its autograd in
float32), `<n>_grad64` (the same network in float64), `<n>_colors` [P, 3] (float32, directions from `<n>_grad`) and
`<n>_colors64` (float64 throughout); `n_uniform` (the first n_uniform points of every net are the uniform ones) and
`weights_sha256` (the digest of trained_weights.npz the nets were loaded from).  Parameters are not stored.
"""
import hashlib
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import outgrads, ref_import  # noqa: E402
from oracle.gen_golden import OUT, load_state, make_args, to_np  # noqa: E402

UNIFORM, NEAR, GRID, ISO, LO, HI = 1000, 1500, 48, 0.0, -1.3, 1.3


def query(kw, net, pts, dirs):
    return kw["network_query_fn"](pts[:, None], dirs, net)[:, 0]


def sigma_and_grad(kw, net, pts, dtype, views):
    x = torch.from_numpy(pts).to(dtype).requires_grad_(True)
    dirs = torch.zeros(len(pts), 3, dtype=dtype) if views else None
    sigma = query(kw, net, x, dirs)[:, 3]
    (g,) = torch.autograd.grad(sigma.sum(), x)
    return to_np(sigma), to_np(g)


def colors(kw, net, pts, grad, dtype, views):
    g = torch.from_numpy(grad).to(dtype)
    n = g.norm(dim=-1, keepdim=True)
    vd = torch.where(n > 0, g / n, torch.zeros_like(g)) if views else None
    with torch.no_grad():
        return to_np(torch.sigmoid(query(kw, net, torch.from_numpy(pts).to(dtype), vd)[:, :3]))


def crossings(kw, net, views, rng):
    """points where the reference's float32 sigma crosses ISO along the edges of a GRID^3 grid (linear interpolation)"""
    a = np.linspace(LO, HI, GRID, dtype=np.float32)
    P = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    with torch.no_grad():
        s = to_np(query(kw, net, torch.from_numpy(P), torch.zeros(len(P), 3) if views else None)[:, 3]).reshape(GRID, GRID, GRID)
    s = s.astype(np.float64)
    P = P.reshape(GRID, GRID, GRID, 3).astype(np.float64)
    out = []
    for ax in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[ax], hi[ax] = slice(0, -1), slice(1, None)
        sa, sb, pa, pb = s[tuple(lo)], s[tuple(hi)], P[tuple(lo)], P[tuple(hi)]
        m = (sa > ISO) != (sb > ISO)
        t = (ISO - sa[m]) / (sb[m] - sa[m])
        out.append(pa[m] + t[:, None] * (pb[m] - pa[m]))
    pts = np.concatenate(out).astype(np.float32)
    if len(pts) > NEAR:
        pts = pts[np.sort(rng.choice(len(pts), NEAR, replace=False))]
    return pts


def main():
    assert ref_import.available(), "reference not found (this script only runs where the reference checkout exists)"
    torch.manual_seed(0)
    torch.set_num_threads(8)
    rn, _ = ref_import.load()
    path = os.path.join(OUT, "trained_weights.npz")
    trained = outgrads.trained_states(path)
    rng = np.random.default_rng(0)
    uniform = rng.uniform(LO, HI, (UNIFORM, 3)).astype(np.float32)
    fx = {"n_uniform": np.int64(UNIFORM),
          "weights_sha256": np.frombuffer(hashlib.sha256(open(path, "rb").read()).digest(), np.uint8)}
    for views in (True, False):
        with tempfile.TemporaryDirectory() as tmp:
            kw, _, _, _, _ = rn.create_nerf(make_args(tmp, use_viewdirs=views, perturb=0.0))
        if views:
            nets = (("c", kw["network_fn"], trained[0]), ("f", kw["network_fine"], trained[1]))
        else:
            nets = (("nv", kw["network_fine"], outgrads.noviews_from_trained(trained[1], 1)),)
        for tag, net, state in nets:
            load_state(net, state)
            pts = np.concatenate([uniform, crossings(kw, net, views, rng)])
            sigma, grad = sigma_and_grad(kw, net, pts, torch.float32, views)
            fx[tag + "_pts"], fx[tag + "_sigma"], fx[tag + "_grad"] = pts, sigma.astype(np.float32), grad.astype(np.float32)
            fx[tag + "_colors"] = colors(kw, net, pts, grad, torch.float32, views).astype(np.float32)
            net.double()
            _, grad64 = sigma_and_grad(kw, net, pts, torch.float64, views)
            fx[tag + "_grad64"] = grad64
            fx[tag + "_colors64"] = colors(kw, net, pts, grad64, torch.float64, views)
            net.float()
            rel = np.linalg.norm(grad - grad64) / np.linalg.norm(grad64)
            print(tag, "points", len(pts), "near", len(pts) - UNIFORM, "grad float32 vs float64 rel-L2 %.3g" % rel)
    np.savez_compressed(os.path.join(OUT, "vertex_attrs.npz"), **fx)


if __name__ == "__main__":
    main()
