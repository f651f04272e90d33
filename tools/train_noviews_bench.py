"""Train-step rates of a network WITHOUT view directions (use_viewdirs=False: output_linear head, output_ch = 5) next to the
view-direction network, on the C2 workload: lego 400x400 rays, N_rand = 4096, 64 + 128 samples, D = 8, W = 256, perturb = 1.

  python tools/train_noviews_bench.py --out DIR [--steps 20] [--warmup 5] [--rounds 3]

Measured in one process on cuda:0, written as JSON to DIR/train_noviews_bench.json with the card's name, power limit and
maximum SM clock (read-only nvidia-smi query):

  * FusedTrainStep (CUDA graph) for both kinds of net, alternated `rounds` times: per round `warmup` steps, then `steps`
    steps each bracketed by CUDA events; the median step time -> rays/s, and the algorithmic rate (FLOP_PER_RAY below);
  * the per-kind kernel split (training-mode forward passes / dgrad chains / wgrad) from nerf_b200_timing_read_kinds over three
    eager steps;
  * the drop-in step a user gets for the no-view net -- render(retraw) + 2 x img2mse + loss.backward() + torch.optim.Adam
    (run_nerf.py:760-784) -- with set_backward('exact') (the fp32 recompute backward) and 'tc'.

Algorithmic work per ray (2 FLOP per MAC of the reference's Linear layers; 256 samples per ray over both passes):
  no view directions, output_ch = 5: fwd 492 288 + wgrad 492 288 + dgrad 460 032 MAC per sample -> 739 639 296 FLOP/ray
  view directions (SURVEY 8d):                                                                      893 190 144 FLOP/ray
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

FLOP_PER_RAY = {"noviews": 739_639_296, "viewdirs": 893_190_144}
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
    ap.add_argument("--out", required=True, help="directory for train_noviews_bench.json (created if missing)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_noviews_bench needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib
    from nerf_pytorch_b200.api import _QueryFn
    from nerf_pytorch_b200.trainer import FusedTrainStep
    from oracle import noviews, synth
    dev = torch.device("cuda:0")
    lib = _lib.load()
    info = gpu_info()
    sb = synth.ray_batch("lego", N_RAYS, seed=0)
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    q = _QueryFn(e, ed, 65536, 10, 4, 0)

    def make_nets(kind):
        nets = []
        for seed in (0, 1):
            if kind == "viewdirs":
                m = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
                st = synth.nerf_state(seed)
            else:
                m = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=0, output_ch=5, skips=[4], use_viewdirs=False)
                st = noviews.nerf_state_noviews(seed)
            m.load_state_dict({k: torch.from_numpy(v) for k, v in st.items()})
            nets.append(m.to(dev))
        return nets

    def kwargs(kind, nets):
        return dict(ndc=False, near=2., far=6., use_viewdirs=kind == "viewdirs", network_fn=nets[0], network_fine=nets[1],
                    network_query_fn=q, N_samples=N_SAMPLES, N_importance=N_IMPORTANCE, perturb=1., white_bkgd=True, raw_noise_std=0.)

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

    # ---- FusedTrainStep, the two kinds alternated ----
    torch.manual_seed(0)
    steppers = {}
    for kind in ("noviews", "viewdirs"):
        tr = FusedTrainStep(sb["H"], sb["W"], sb["K"], N_RAYS, kwargs(kind, make_nets(kind)), lrate=5e-4, lrate_decay=250)
        tr.rays.copy_(rays_dev); tr.target.copy_(tgt_dev)
        steppers[kind] = tr
    times = {k: [] for k in steppers}
    for _ in range(args.rounds):
        for kind, tr in steppers.items():
            times[kind] += timed(tr.step_device, args.steps, args.warmup)
    fused = {}
    for kind, tr in steppers.items():
        ms = float(np.median(times[kind]))
        lib.nerf_b200_timing_enable(1)
        for _ in range(3):
            tr._pack_rays(); tr._fwd_bwd(); tr._adam()
        torch.cuda.synchronize()
        kms, kn, kfl = C.c_double(), C.c_int64(), C.c_double()
        kinds = (C.c_double * 3)()
        lib.nerf_b200_timing_read_kinds(C.byref(kms), C.byref(kn), C.byref(kfl), kinds)
        lib.nerf_b200_timing_enable(0)
        fused[kind] = {"ms_per_step_median": ms, "ms_per_step_min": float(np.min(times[kind])), "ms_per_step_max": float(np.max(times[kind])),
                       "steps_timed": len(times[kind]), "rays_per_s": N_RAYS / (ms * 1e-3),
                       "flop_per_ray": FLOP_PER_RAY[kind], "algorithmic_tflops": N_RAYS * FLOP_PER_RAY[kind] / (ms * 1e-3) / 1e12,
                       "loss_last_step": float(tr.state[0].item()),
                       "kernel_ms_per_step_eager": {"forward_passes_training_mode": kinds[0] / 3, "dgrad_chains": kinds[1] / 3, "wgrad": kinds[2] / 3}}
    del steppers
    torch.cuda.empty_cache()

    # ---- the drop-in step of the no-view net: render + 2 x img2mse + backward + Adam, exact vs tensor-core backward ----
    dropin = {}
    for mode in ("exact", "tc", "exact", "tc"):
        nets = make_nets("noviews")
        opt = torch.optim.Adam([p for n in nets for p in n.parameters()], lr=5e-4, betas=(0.9, 0.999))
        kw = kwargs("noviews", nets)
        nb.set_backward(mode)

        def step():
            rgb, _, _, ex = nb.render(sb["H"], sb["W"], sb["K"], chunk=32768, rays=rays_dev, retraw=True, **kw)
            opt.zero_grad()
            loss = nb.img2mse(rgb, tgt_dev) + nb.img2mse(ex["rgb0"], tgt_dev)
            loss.backward()
            opt.step()
        try:
            dropin.setdefault(mode, []).extend(timed(step, args.steps, args.warmup))
        finally:
            nb.set_backward("tc")
    drop = {m: {"ms_per_step_median": float(np.median(v)), "rays_per_s": N_RAYS / (float(np.median(v)) * 1e-3), "steps_timed": len(v)}
            for m, v in dropin.items()}
    res = {"gpu": info, "workload": f"lego 400x400, N_rand={N_RAYS}, {N_SAMPLES}+{N_IMPORTANCE} samples, D=8 W=256, perturb=1, white_bkgd",
           "fused_train_step": fused, "dropin_step_noviews": drop,
           "notes": "fused_train_step: FusedTrainStep.step_device (CUDA-graph replay incl. ray packing and Adam), CUDA events per step, "
                    "the two kinds alternated; kernel split from an eager pass with events around each launch. dropin: render(retraw) "
                    "+ 2 x img2mse + loss.backward() + torch.optim.Adam.step(), CUDA events per step."}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "train_noviews_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
