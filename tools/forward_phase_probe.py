"""Where march_wg_kernel's time goes, per pass, at bench.py's forward shape (4096 lego rays, 64 + 128 samples, D = 8 W = 256 with
view directions): an experiments build of libnerf_b200.so (-DNERF_B200_PHASE_PROBE, compiled into a temporary directory
unless --lib names one) in which thread 0 of each MMA warpgroup adds up clock64 time per phase (fused_wg.cuh: Phases):
  full        waiting on a weight-ring stage's full barrier
  gap         from the end of a layer's MMAs (wgmma_wait<0>) to the next layer's first full wait, inside a tile: epilogue + bias
  sampler     from a tile's start to its first layer: pts = o + d z and the positional encoding
  compositor  from a tile's last layer to its end: heads, raw rows, compositing
  total       the warpgroup's whole run
Prints one JSON line per pass (coarse, fine) and MMA warpgroup: clocks per CTA and launch (mean over CTAs) and each phase's share
of the total.  The product library is never touched."""
import argparse, ctypes as C, json, os, subprocess, sys, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def build_probe_lib(out_dir):
    import __graft_entry__ as ge
    lib = os.path.join(out_dir, "libnerf_b200_phase_probe.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc] + ge.NVCC_FLAGS + ["-DNERF_B200_PHASE_PROBE", "-o", lib, os.path.join(ge.CSRC, "capi.cu")], check=True, cwd=ge.CSRC)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="a library built with -DNERF_B200_PHASE_PROBE (default: build one in a temporary directory)")
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    tmp = tempfile.TemporaryDirectory()
    path = args.lib or build_probe_lib(tmp.name)
    import torch
    from nerf_pytorch_b200 import _lib
    _lib.LIB_PATH = path                             # the experiments build serves this process
    lib = _lib.load()
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.api import _QueryFn
    from oracle import synth
    assert torch.cuda.is_available(), "the phase probe needs a GPU"
    dev = torch.device("cuda:0")
    for name in ("nerf_b200_phase_probe_reset", "nerf_b200_phase_probe_read", "nerf_b200_phase_probe_shape"):
        getattr(lib, name).restype = C.c_int
    lib.nerf_b200_phase_probe_read.argtypes = [C.c_void_p, C.c_size_t]
    slots, ctas, nph = C.c_int(), C.c_int(), C.c_int()
    lib.nerf_b200_phase_probe_shape(C.byref(slots), C.byref(ctas), C.byref(nph))

    nets = []
    for seed in (0, 1):
        m = nb.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.nerf_state(seed).items()})
        nets.append(m.to(dev))
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    q = _QueryFn(e, ed, 65536, 10, 4, 0)
    sb = synth.ray_batch("lego", 4096, seed=0)
    rays = torch.from_numpy(sb["rays"]).to(dev)
    kw = dict(ndc=False, near=2., far=6., use_viewdirs=True, network_fn=nets[0], network_fine=nets[1], network_query_fn=q,
              N_samples=64, N_importance=128, perturb=0., white_bkgd=True, raw_noise_std=0.)

    def step():
        with torch.no_grad():
            nb.render(sb["H"], sb["W"], sb["K"], chunk=32768, rays=rays, **kw)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    _lib.check(lib.nerf_b200_phase_probe_reset(), "phase_probe_reset")
    for _ in range(args.steps):
        step()
    tab = np.zeros((slots.value, ctas.value, 2, nph.value), dtype=np.uint64)
    _lib.check(lib.nerf_b200_phase_probe_read(tab.ctypes.data, tab.nbytes), "phase_probe_read")
    names = ["full", "gap", "sampler", "compositor", "total"]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "steps": args.steps}), flush=True)
    for slot, pas in enumerate(("coarse", "fine")):
        used = tab[slot, :, 0, 4] > 0
        for w in range(2):
            per = tab[slot, used, w, :].astype(np.float64) / args.steps
            mean = per.mean(axis=0)
            print(json.dumps({"pass": pas, "warpgroup": w + 1, "ctas": int(used.sum()),
                              "clocks_per_cta": {n: round(float(v)) for n, v in zip(names, mean)},
                              "share": {n: round(float(v / mean[4]), 4) for n, v in zip(names[:4], mean[:4])}}), flush=True)


if __name__ == "__main__":
    main()
