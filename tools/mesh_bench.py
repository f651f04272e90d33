"""Mesh extraction on one GPU: density_grid against the extraction notebook's way, and marching cubes.

    python tools/mesh_bench.py --out DIR [--reps 5] [--sizes 256 512]

The network is the trained fine net of tests/golden/trained_weights.npz (8 x 256, view directions).  Per grid size n (an n^3 grid
over [-1.3, 1.3]^3) and tensor-core precision:

  * density_grid: points/s of nerf_pytorch_b200.density_grid;
  * notebook: points/s of the original release's extraction notebook on this library -- the [n^3, 3] points materialised with
    meshgrid, run_network on 65 536-point chunks with zero view directions, sigma = raw[..., 3];
  * both arms alternate in the same process, 3 rounds of --reps runs each after a warm-up; medians of CUDA-event times;
  * peak torch.cuda.max_memory_allocated above the resident network of each arm;
  * whether the two sigma grids are equal bit for bit;
  * marching cubes (count, one host sync, emit) on density_grid's sigma at iso 10: time, V and F.

The card's name and power limit are read in the same run.  Writes DIR/mesh_bench.json and prints it."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CHUNK = 65536
ISO = 10.0


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = (s.strip() for s in q.split(","))
    except Exception as e:                                   # the measurement stands; the card facts are then missing
        out["nvidia_smi_error"] = str(e)
    return out


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench: no CUDA device (the numbers are GPU measurements; there is no CPU fallback)")
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.api import _QueryFn
    w = np.load(os.path.join(ROOT, "tests", "golden", "trained_weights.npz"))
    net = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
    net.load_state_dict({k[2:]: torch.from_numpy(w[k]) for k in w.files if k.startswith("f.")})
    net = net.cuda()
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    q = _QueryFn(e, ed, CHUNK, 10, 4, 0)
    res = {"card": card(), "net": "trained fine net, 8 x 256, view directions", "chunk": CHUNK, "iso": ISO, "reps": args.reps, "runs": {}}

    def notebook(xs):
        pts = torch.stack(torch.meshgrid(xs, xs, xs, indexing="ij"), -1).reshape(-1, 3)
        sigma = torch.empty(pts.shape[0], device=pts.device)
        zeros = torch.zeros((CHUNK, 3), device=pts.device)
        with torch.no_grad():
            for i in range(0, pts.shape[0], CHUNK):
                p = pts[i:i + CHUNK]
                sigma[i:i + CHUNK] = nb.run_network(p.reshape(-1, 1, 3), zeros[:p.shape[0]], net, e, ed)[:, 0, 3]
        return sigma.reshape(len(xs), len(xs), len(xs))

    for n in args.sizes:
        xs = torch.linspace(-1.3, 1.3, n, device="cuda")
        P = n ** 3
        for prec in ("tc_fp16", "tc_split"):
            nb.set_precision(prec)
            arms = {"density_grid": lambda: nb.density_grid(net, q, xs, xs, xs), "notebook": lambda: notebook(xs)}
            peak = {}
            out = {}
            for k, fn in arms.items():                       # warm-up, and each arm's peak memory on its own
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                out[k] = fn()
                torch.cuda.synchronize()
                peak[k] = torch.cuda.max_memory_allocated() - base
                if k == "notebook":
                    del out[k]
            ref = notebook(xs)
            same = bool(torch.equal(out["density_grid"].view(torch.int32), ref.view(torch.int32)))
            del ref
            ms = {k: [] for k in arms}
            for _ in range(3):
                for _ in range(args.reps):
                    for k, fn in arms.items():
                        t, r = timed(fn)
                        ms[k].append(t)
                        del r
            med = {k: float(np.median(v)) for k, v in ms.items()}
            sigma = out.pop("density_grid")
            mc_ms, (v, f) = [], (None, None)
            for _ in range(args.reps + 1):
                t, (v, f) = timed(lambda: nb.marching_cubes(sigma, xs, xs, xs, ISO))
                mc_ms.append(t)
            run = {"points": P, "bit_identical": same,
                   "density_grid_ms": med["density_grid"], "notebook_ms": med["notebook"],
                   "density_grid_points_per_s": P / med["density_grid"] * 1e3, "notebook_points_per_s": P / med["notebook"] * 1e3,
                   "speedup": med["notebook"] / med["density_grid"],
                   "peak_bytes": peak, "ms_all": ms,
                   "marching_cubes_ms": float(np.median(mc_ms[1:])), "V": int(v.shape[0]), "F": int(f.shape[0])}
            res["runs"][f"{n}^3 {prec}"] = run
            del sigma, v, f
            torch.cuda.empty_cache()
            print(f"{n}^3 {prec}: density_grid {run['density_grid_ms']:.1f} ms ({run['density_grid_points_per_s'] / 1e9:.3f} Gpts/s), "
                  f"notebook {run['notebook_ms']:.1f} ms ({run['notebook_points_per_s'] / 1e9:.3f} Gpts/s), x{run['speedup']:.2f}, "
                  f"peak {peak['density_grid'] / 2**30:.2f} / {peak['notebook'] / 2**30:.2f} GiB, bit-identical {same}, "
                  f"marching cubes {run['marching_cubes_ms']:.1f} ms (V {run['V']}, F {run['F']})", flush=True)
    nb.set_precision("tc_fp16")
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "mesh_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}))


if __name__ == "__main__":
    main()
