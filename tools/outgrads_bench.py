"""Cost of a loss that reads more than rgb_map, on the drop-in training step: C2 workload (lego 400x400 rays, N_rand = 4096,
64 + 128 samples, view directions, perturb = 1), render(retraw) + loss + loss.backward() + torch.optim.Adam (run_nerf.py:760-784)
with the tensor-core backward.

  python tools/outgrads_bench.py --out DIR [--steps 20] [--warmup 5] [--rounds 3]

Two losses, alternated `rounds` times in one process (per round `warmup` untimed steps, then `steps` steps each bracketed by
CUDA events; median step time -> rays/s):

  rgb: img2mse(rgb) + img2mse(rgb0)                                   (nerf_b200_render_rays_bwd_tc)
  all: rgb + L_acc + 0.1 L_disp + 1e-3 L_raw (oracle/outgrads.loss_of) (nerf_b200_render_rays_bwd_tc_outs)

Written as JSON to DIR/outgrads_bench.json with the card's name, power limit and maximum SM clock (read-only nvidia-smi query).
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
    ap.add_argument("--out", required=True, help="directory for outgrads_bench.json (created if missing)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("outgrads_bench needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.api import _QueryFn
    from oracle import outgrads, synth
    dev = torch.device("cuda:0")
    info = gpu_info()
    sb = synth.ray_batch("lego", N_RAYS, seed=0)
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    q = _QueryFn(e, ed, 65536, 10, 4, 0)
    nets = []
    for seed in (0, 1):
        m = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.nerf_state(seed).items()})
        nets.append(m.to(dev))
    opt = torch.optim.Adam(list(nets[0].parameters()) + list(nets[1].parameters()), lr=5e-4, betas=(0.9, 0.999))
    rays = torch.from_numpy(sb["rays"]).to(dev)
    rng = np.random.default_rng(0)
    target = torch.from_numpy(rng.random((N_RAYS, 3), dtype=np.float32)).to(dev)
    t_acc = torch.from_numpy(rng.random(N_RAYS, dtype=np.float32)).to(dev)
    kw = dict(ndc=False, near=2., far=6., use_viewdirs=True, network_fn=nets[0], network_fine=nets[1], network_query_fn=q,
              N_samples=N_SAMPLES, N_importance=N_IMPORTANCE, perturb=1., white_bkgd=True, raw_noise_std=0., retraw=True)

    def step(which):
        rgb, disp, acc, ex = nb.render(400, 400, sb["K"], chunk=32768, rays=rays, **kw)
        if which == "rgb":
            loss = nb.img2mse(rgb, target) + nb.img2mse(ex["rgb0"], target)
        else:
            loss = outgrads.loss_of("all", rgb, disp, acc, ex, target, t_acc)
        opt.zero_grad()
        loss.backward()
        opt.step()

    times = {"rgb": [], "all": []}
    for _ in range(args.rounds):
        for which in ("rgb", "all"):
            for _ in range(args.warmup):
                step(which)
            torch.cuda.synchronize()
            for _ in range(args.steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                step(which)
                b.record()
                b.synchronize()
                times[which].append(a.elapsed_time(b))
    res = {"gpu": info, "workload": f"lego {N_RAYS} rays x {N_SAMPLES}+{N_IMPORTANCE}, view directions, perturb 1, tensor-core backward",
           "rounds": args.rounds, "steps": args.steps, "warmup": args.warmup}
    for which, t in times.items():
        med = float(np.median(t))
        res[which] = {"median_ms": med, "min_ms": float(np.min(t)), "rays_per_s": N_RAYS / (med * 1e-3)}
    res["all_over_rgb"] = res["all"]["median_ms"] / res["rgb"]["median_ms"]
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "outgrads_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
