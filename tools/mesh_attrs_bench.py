"""Vertex attributes on one GPU: the cost of density_gradient and vertex_attributes beside the mesh extraction they follow, and how
far the grid's central-difference normals are from the network's own.

    python tools/mesh_attrs_bench.py --out DIR [--reps 5] [--sizes 256 512]

The network is the trained fine net of tests/golden/trained_weights.npz (8 x 256, view directions, multires 10), the settings of
tools/mesh_bench.py: an n^3 grid over [-1.3, 1.3]^3, iso 10, precision tc_fp16.  Per grid size n:

  * the median CUDA-event time of density_grid, marching_cubes (count, one host sync, emit), density_gradient on the mesh's
    vertices and vertex_attributes (density_gradient, then run_network for the colours), the four alternated in one process,
    3 rounds of --reps runs each after a warm-up;
  * the angle between each vertex's analytic normal (-grad / |grad|) and the grid's: central differences of the same sigma grid
    (torch.gradient: one-sided at the border) at the two ends of the vertex's grid edge, interpolated along the edge as
    marching_cubes places the vertex, then negated and normalised.  Median and 95th percentile, in degrees.

The card's name and power limit are read in the same run.  Writes DIR/mesh_attrs_bench.json and prints it."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from mesh_bench import card, timed  # noqa: E402

ISO = 10.0


def grid_normals(sigma, xs, verts):
    """the central-difference normal of sigma [n, n, n] on the uniform axis xs, interpolated along each vertex's grid edge"""
    n = len(xs)
    inside = sigma > ISO
    act = torch.zeros(sigma.shape + (3,), dtype=torch.bool, device=sigma.device)
    act[:-1, :, :, 0] = inside[:-1] != inside[1:]
    act[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    act[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    idx = torch.nonzero(act)                          # vertex ids follow the crossing edges in C order, then axis
    del act, inside
    assert len(idx) == len(verts)
    lo, ax = idx[:, :3], idx[:, 3]
    hi = lo + torch.eye(3, dtype=lo.dtype, device=lo.device)[ax]
    h = float(xs[1] - xs[0])
    g = torch.stack(torch.gradient(sigma, spacing=h), -1)
    ga, gb = g[lo[:, 0], lo[:, 1], lo[:, 2]], g[hi[:, 0], hi[:, 1], hi[:, 2]]
    del g
    rows = torch.arange(len(verts), device=verts.device)
    ca, cb = xs[lo[rows, ax]], xs[hi[rows, ax]]
    t = ((verts[rows, ax] - ca) / (cb - ca))[:, None]
    gv = ga + t * (gb - ga)
    assert int(hi.max()) < n
    return -gv / gv.norm(dim=-1, keepdim=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_attrs_bench: no CUDA device (the numbers are GPU measurements; there is no CPU fallback)")
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.api import _QueryFn
    w = np.load(os.path.join(ROOT, "tests", "golden", "trained_weights.npz"))
    net = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
    net.load_state_dict({k[2:]: torch.from_numpy(w[k]) for k in w.files if k.startswith("f.")})
    net = net.cuda()
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    q = _QueryFn(e, ed, 65536, 10, 4, 0)
    nb.set_precision("tc_fp16")
    res = {"card": card(), "net": "trained fine net, 8 x 256, view directions", "iso": ISO, "precision": "tc_fp16",
           "reps": args.reps, "runs": {}}
    for n in args.sizes:
        xs = torch.linspace(-1.3, 1.3, n, device="cuda")
        sigma = nb.density_grid(net, q, xs, xs, xs)
        v, f = nb.marching_cubes(sigma, xs, xs, xs, ISO)
        arms = {"density_grid": lambda: nb.density_grid(net, q, xs, xs, xs),
                "marching_cubes": lambda: nb.marching_cubes(sigma, xs, xs, xs, ISO),
                "density_gradient": lambda: nb.density_gradient(net, q, v),
                "vertex_attributes": lambda: nb.vertex_attributes(net, q, v)}
        for fn in arms.values():                          # warm-up
            fn()
        ms = {k: [] for k in arms}
        for _ in range(3):
            for _ in range(args.reps):
                for k, fn in arms.items():
                    t, r = timed(fn)
                    ms[k].append(t)
                    del r
        med = {k: float(np.median(x)) for k, x in ms.items()}
        normals, _ = nb.vertex_attributes(net, q, v)
        ng = grid_normals(sigma, xs, v)
        ok = (normals.norm(dim=-1) > 0) & torch.isfinite(ng).all(-1)
        ang = torch.rad2deg(torch.acos((normals[ok].double() * ng[ok].double()).sum(-1).clamp(-1, 1))).cpu().numpy()
        run = {"V": int(v.shape[0]), "F": int(f.shape[0]), "ms": med, "ms_all": ms, "spacing": float(xs[1] - xs[0]),
               "angle_deg_median": float(np.median(ang)), "angle_deg_p95": float(np.percentile(ang, 95)),
               "angle_vertices": int(len(ang)), "zero_normals": int((~ok).sum())}
        res["runs"][f"{n}^3"] = run
        print(f"{n}^3: V {run['V']}, F {run['F']}; " + ", ".join(f"{k} {t:.2f} ms" for k, t in med.items()) +
              f"; grid vs analytic normal: median {run['angle_deg_median']:.2f} deg, p95 {run['angle_deg_p95']:.2f} deg", flush=True)
        del sigma, v, f, normals, ng
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "mesh_attrs_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}))


if __name__ == "__main__":
    main()
