"""Train-step rates of precision tc_split with the split backward (set_backward('tc_split')) next to its alternatives, on BASELINE
config 2 with view directions: lego 400x400 rays, N_rand = 4096, 64 + 128 samples, D = 8, W = 256, perturb = 1.

  python tools/split_train_bench.py --out DIR [--steps 10] [--warmup 3] [--rounds 3]

Measured in one process on cuda:0, written as JSON to DIR/split_train_bench.json with the card's name, power limit and maximum SM
clock (read-only nvidia-smi query).  Arms, alternated `rounds` times, each `warmup` steps then `steps` steps bracketed by CUDA
events (median):

  * fused_tc_fp16:    FusedTrainStep on tc_fp16 (one CUDA graph: pack, training forward, MSE seeds, backward, Adam);
  * fused_split:      FusedTrainStep on tc_split with set_backward('tc_split') (the split image, records and backward in the graph);
  * dropin_tc_fp16:   render(retraw) + 2 x img2mse + loss.backward() + torch.optim.Adam on tc_fp16, set_backward('tc');
  * dropin_split_exact: the same step on tc_split with the exact fp32 recompute backward (what tc_split trained with before);
  * dropin_split:     the same step on tc_split with set_backward('tc_split').

Per arm: the kernel split by kind (nerf_b200_timing_read_kinds: forward passes / dgrad chains / wgrad) over three eager steps, and
for the drop-in arms the peak memory of one step (torch.cuda.max_memory_allocated).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_RAYS, N_SAMPLES, N_IMPORTANCE = 4096, 64, 128


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
    ap.add_argument("--out", required=True, help="directory for split_train_bench.json (created if missing)")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("split_train_bench needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib
    from nerf_pytorch_b200.api import _QueryFn
    from nerf_pytorch_b200.trainer import FusedTrainStep
    from oracle import synth
    dev = torch.device("cuda:0")
    lib = _lib.load()
    info = gpu_info()
    sb = synth.ray_batch("lego", N_RAYS, seed=0)
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    q = _QueryFn(e, ed, 65536, 10, 4, 0)

    def make_nets():
        nets = []
        for seed in (0, 1):
            m = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
            m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.nerf_state(seed).items()})
            nets.append(m.to(dev))
        return nets

    def kwargs(nets):
        return dict(ndc=False, near=2., far=6., use_viewdirs=True, network_fn=nets[0], network_fine=nets[1], network_query_fn=q,
                    N_samples=N_SAMPLES, N_importance=N_IMPORTANCE, perturb=1., white_bkgd=True, raw_noise_std=0.)

    rays_dev = torch.from_numpy(sb["rays"]).to(dev)
    tgt_dev = torch.rand(N_RAYS, 3, generator=torch.Generator().manual_seed(1)).to(dev)

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()
            ts.append((a, b))
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in ts]

    modes = {"dropin_tc_fp16": ("tc_fp16", "tc"), "dropin_split_exact": ("tc_split", "exact"), "dropin_split": ("tc_split", "tc_split")}
    arms = {}
    for name, (prec, bwd) in modes.items():
        nets = make_nets()
        opt = torch.optim.Adam([p for n in nets for p in n.parameters()], lr=5e-4, betas=(0.9, 0.999))
        kw = kwargs(nets)

        def step(kw=kw, opt=opt, prec=prec, bwd=bwd):
            nb.set_precision(prec)
            nb.set_backward(bwd)
            try:
                rgb, _, _, ex = nb.render(sb["H"], sb["W"], sb["K"], chunk=32768, rays=rays_dev, retraw=True, **kw)
                opt.zero_grad()
                loss = nb.img2mse(rgb, tgt_dev) + nb.img2mse(ex["rgb0"], tgt_dev)
                loss.backward()
                opt.step()
            finally:
                nb.set_precision("tc_fp16")
                nb.set_backward("tc")
        arms[name] = step
    fused = {}
    for name, (prec, bwd) in (("fused_tc_fp16", ("tc_fp16", "tc")), ("fused_split", ("tc_split", "tc_split"))):
        torch.manual_seed(0)
        nb.set_precision(prec)
        nb.set_backward(bwd)
        try:
            tr = FusedTrainStep(sb["H"], sb["W"], sb["K"], N_RAYS, kwargs(make_nets()), lrate=5e-4, lrate_decay=250)
        finally:
            nb.set_precision("tc_fp16")
            nb.set_backward("tc")
        tr.rays.copy_(rays_dev); tr.target.copy_(tgt_dev)
        arms[name] = tr.step_device
        fused[name] = tr

    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            times[name] += timed(fn, args.steps, args.warmup)
    res_arms = {}
    for name, fn in arms.items():
        ms = float(np.median(times[name]))
        r = {"ms_per_step_median": ms, "ms_per_step_min": float(np.min(times[name])), "ms_per_step_max": float(np.max(times[name])),
             "steps_timed": len(times[name]), "rays_per_s": N_RAYS / (ms * 1e-3)}
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        lib.nerf_b200_timing_enable(1)
        for _ in range(3):
            if name in fused:                   # the graph's work, eagerly, with events around each launch
                tr = fused[name]
                tr._pack_rays(); tr._fwd_bwd(); tr._adam()
            else:
                fn()
        torch.cuda.synchronize()
        kms, kn, kfl = C.c_double(), C.c_int64(), C.c_double()
        kinds = (C.c_double * 3)()
        lib.nerf_b200_timing_read_kinds(C.byref(kms), C.byref(kn), C.byref(kfl), kinds)
        lib.nerf_b200_timing_enable(0)
        r["kernel_ms_per_step_eager"] = {"forward_passes": kinds[0] / 3, "dgrad_chains": kinds[1] / 3, "wgrad": kinds[2] / 3}
        if name not in fused:
            r["peak_memory_gib"] = torch.cuda.max_memory_allocated() / 2**30
        res_arms[name] = r
    res = {"gpu": info, "workload": f"lego 400x400, N_rand={N_RAYS}, {N_SAMPLES}+{N_IMPORTANCE} samples, D=8 W=256, view directions, perturb=1, white_bkgd",
           "arms": res_arms,
           "speedup_fused_split_vs_split_exact": res_arms["dropin_split_exact"]["ms_per_step_median"] / res_arms["fused_split"]["ms_per_step_median"],
           "speedup_split_vs_split_exact": res_arms["dropin_split_exact"]["ms_per_step_median"] / res_arms["dropin_split"]["ms_per_step_median"],
           "notes": "CUDA events per step, the arms alternated; kernel split from eager steps with events around each launch "
                    "(forward passes in training mode when a backward follows)."}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "split_train_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
