"""What a FusedTrainStep step of fewer rays than its capacity costs: the first use of a new size (its capture) and the replay
of the short step next to the full one.  Workload: lego 400x400 rays, N_rand = 1024 with the 816-ray last batch of an epoch
(fern at factor 8 / llffhold 8), 64 + 128 samples, D = 8, W = 256 with view directions, perturb = 1, raw_noise_std = 1.

  python tools/variable_batch_time.py --out DIR [--capacity 1024] [--short 816] [--steps 20] [--rounds 3]

Measured in one process on cuda:0 and written as JSON to DIR/variable_batch_time.json, with the card's name, power limit and
maximum SM clock read in the same run (read-only nvidia-smi query):

  * first_use: host wall clock of the first step_device(n_rays=short) (two eager warm-up steps, the capture, the step; the
    device synchronised before and after), and torch.cuda.memory_allocated() before and after it;
  * replay: CUDA events around each step_device of `steps` steps per size, the two sizes alternated `rounds` times; median per
    size and the rate in rays/s;
  * grow: the same first-use numbers for a size below the capacity whose tile plan needs more record or workspace bytes than
    the capacity's (the largest such size), which gets buffers of its own.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    ap.add_argument("--out", required=True, help="directory for variable_batch_time.json (created if missing)")
    ap.add_argument("--capacity", type=int, default=1024)
    ap.add_argument("--short", type=int, default=816)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("variable_batch_time needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.api import _QueryFn
    from nerf_pytorch_b200.trainer import FusedTrainStep
    from oracle import synth
    dev = torch.device("cuda:0")
    info = gpu_info()
    cap, short = args.capacity, args.short
    sb = synth.ray_batch("lego", cap, seed=0)
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    nets = []
    for seed in (0, 1):
        m = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.nerf_state(seed).items()})
        nets.append(m.to(dev))
    kw = dict(ndc=False, near=2., far=6., use_viewdirs=True, network_fn=nets[0], network_fine=nets[1], network_query_fn=_QueryFn(e, ed, 65536, 10, 4, 0),
              N_samples=64, N_importance=128, perturb=1., white_bkgd=True, raw_noise_std=1.)
    torch.manual_seed(0)
    tr = FusedTrainStep(sb["H"], sb["W"], sb["K"], cap, kw, lrate=5e-4, lrate_decay=250)
    tr.rays.copy_(torch.from_numpy(sb["rays"]).to(dev))
    tr.target.copy_(torch.rand(cap, 3, generator=torch.Generator().manual_seed(1)).to(dev))
    for _ in range(args.warmup):
        tr.step_device()

    def first_use(n):
        torch.cuda.synchronize()
        mem0 = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        tr.step_device(n_rays=n)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        return {"n_rays": n, "ms_first_step": ms, "memory_allocated_before": mem0, "memory_allocated_after": torch.cuda.memory_allocated()}

    first = first_use(short)

    def timed(n):
        for _ in range(args.warmup):
            tr.step_device(n_rays=n)
        ev = []
        for _ in range(args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); tr.step_device(n_rays=n); b.record()
            ev.append((a, b))
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in ev]
    times = {cap: [], short: []}
    for _ in range(args.rounds):
        for n in (cap, short):
            times[n] += timed(n)
    replay = {str(n): {"ms_per_step_median": float(np.median(t)), "ms_per_step_min": float(np.min(t)), "ms_per_step_max": float(np.max(t)),
                       "steps_timed": len(t), "rays_per_s": n / (float(np.median(t)) * 1e-3)} for n, t in times.items()}

    # a size whose plan needs more than the capacity's records or workspaces
    lib, Sc, Sf = tr.lib, tr.Sc, tr.Sc + tr.Ni
    have = {k: tr._sized[cap][k].numel() for k in ("act_c", "mask_c", "act_f", "mask_f", "ws", "bws")}

    def needs(n):
        out = {}
        for tag, S, np_ in (("c", Sc, tr._np_c), ("f", Sf, tr._np_f)):
            ab, mb = C.c_size_t(0), C.c_size_t(0)
            lib.nerf_b200_train_record_bytes(n, S, C.byref(np_), C.byref(ab), C.byref(mb))
            out["act_" + tag], out["mask_" + tag] = ab.value, mb.value
        out["ws"] = lib.nerf_b200_march_workspace_bytes(n, Sf)
        out["bws"] = lib.nerf_b200_render_rays_bwd_tc_workspace_bytes(n, Sc, C.byref(tr._np_c), Sf, C.byref(tr._np_f)) + 1024
        return out
    grow = next((n for n in range(cap - 1, 0, -1) if n != short and any(v > have[k] for k, v in needs(n).items())), None)
    grow_res = None
    if grow is not None:
        grow_res = first_use(grow)
        grow_res["buffers_above_capacity"] = {k: [v, have[k]] for k, v in needs(grow).items() if v > have[k]}
    res = {"gpu": info,
           "workload": f"lego 400x400, capacity {cap} rays, short batch {short} rays, 64+128 samples, D=8 W=256 + view head, perturb=1, raw_noise_std=1",
           "first_use": first, "replay": replay, "grow": grow_res,
           "notes": "first_use: host wall clock of the first step_device(n_rays) at that size with the device synchronised before and after "
                    "(two eager warm-up steps + the capture + one replayed step). replay: CUDA events around step_device (ray packing + graph "
                    "replay), the sizes alternated; median over rounds x steps."}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "variable_batch_time.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
