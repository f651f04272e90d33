"""Forward time of the three precisions on BASELINE config 2: 4096 lego rays, 64 + 128 samples, 8 x 256 networks with view
directions, render() under torch.no_grad() on device-resident rays.

  python tools/precision_bench.py [--out DIR] [--steps 20] [--warmup 5] [--rounds 3]

tc_fp16, tc_split and fp32 alternate `rounds` times in one process.  Per round and precision: `warmup` untimed renders, then
`steps` renders, each after a 256 MB write that flushes L2 and bracketed by CUDA events.  Reported: the median step time over
all rounds, rays/s, and each precision's rgb_map distance from fp32's on the same rays.  The card's name, power limit and
maximum SM clock come from a read-only nvidia-smi query in the same run.  Prints one JSON line; with --out also writes it to
DIR/precision_bench.json.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_RAYS, N_SAMPLES, N_IMPORTANCE = 4096, 64, 128
MODES = ("tc_fp16", "tc_split", "fp32")


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power, clk = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:                     # the numbers are still measured; the card is then unnamed
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("precision_bench needs a CUDA device")
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.api import _QueryFn
    from oracle import synth
    dev = torch.device("cuda:0")
    sb = synth.ray_batch("lego", N_RAYS, seed=0)
    nets = []
    for seed in (0, 1):
        m = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.nerf_state(seed).items()})
        nets.append(m.to(dev))
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    kw = dict(chunk=32768, rays=torch.from_numpy(sb["rays"]).to(dev), ndc=False, near=2., far=6., use_viewdirs=True,
              network_fn=nets[0], network_fine=nets[1], network_query_fn=_QueryFn(e, ed, 65536, 10, 4, 0),
              N_samples=N_SAMPLES, N_importance=N_IMPORTANCE, perturb=0., white_bkgd=True, raw_noise_std=0.)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def render():
        with torch.no_grad():
            return nb.render(sb["H"], sb["W"], sb["K"], **kw)[0]

    times = {m: [] for m in MODES}
    rgb = {}
    try:
        for _ in range(a.rounds):
            for mode in MODES:
                nb.set_precision(mode)
                for _ in range(a.warmup):
                    rgb[mode] = render()
                for _ in range(a.steps):
                    flush.fill_(1)
                    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    t0.record()
                    render()
                    t1.record()
                    t1.synchronize()
                    times[mode].append(t0.elapsed_time(t1))
    finally:
        nb.set_precision("tc_fp16")
    ref = rgb["fp32"].double()
    res = {"workload": f"render, {N_RAYS} lego rays, {N_SAMPLES} + {N_IMPORTANCE} samples, 8x256 with view directions, no_grad",
           "gpu": gpu_info(), "steps": a.steps * a.rounds}
    for mode in MODES:
        ms = float(np.median(times[mode]))
        res[mode] = {"ms_median": ms, "ms_min": float(np.min(times[mode])), "ms_max": float(np.max(times[mode])),
                     "rays_per_s": N_RAYS / ms * 1e3,
                     "rgb_map_rel_l2_vs_fp32": float((rgb[mode].double() - ref).norm() / ref.norm())}
    res["fp32_over_tc_split"] = res["fp32"]["ms_median"] / res["tc_split"]["ms_median"]
    res["tc_split_over_tc_fp16"] = res["tc_split"]["ms_median"] / res["tc_fp16"]["ms_median"]
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "precision_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
