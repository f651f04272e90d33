"""Per-SM HBM streaming rates of the copy mechanisms the training kernels can use (libnerf_b200_dev.so: dram_stream_probe_kernel):
cp.async.bulk global->shared rings, 16-byte cp.async rings, cp.async.bulk shared->global, plain vector loads / stores.
One CTA per SM, disjoint 16 MiB regions per CTA and launch (8 launches walk a 19 GB buffer: nothing is re-read from L2).
Prints JSON lines: mechanism, ring, CTAs, TB/s (CUDA events) and bytes/clock/SM (clock64 inside the kernel, median CTA)."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nerf_pytorch_b200 import _lib
dev = torch.device("cuda:0")
lib = _lib.load_dev()
per = 16 << 20
nb_max = torch.cuda.get_device_properties(0).multi_processor_count
buf = torch.zeros(8 * nb_max * per, dtype=torch.uint8, device=dev)
out = torch.zeros(nb_max + 8, dtype=torch.int64, device=dev)
st = torch.cuda.current_stream().cuda_stream
names = {0: "cp.async.bulk g2s", 1: "cp.async 16B g2s", 2: "cp.async.bulk s2g", 3: "st.global.v4", 4: "ld.global.v4"}
def run(mode, chunk, stages, nblk, scatter=0):
    best, cyc = 1e9, None
    for rep in range(8):
        off = rep * nb_max * per
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check_dev(lib.nerf_b200_debug_dram_stream(buf.data_ptr() + off, per, chunk, stages, mode, nblk, scatter, out.data_ptr(), st), "dram_stream")
        e1.record(); torch.cuda.synchronize()
        if rep >= 2 and e0.elapsed_time(e1) < best:
            best = e0.elapsed_time(e1); cyc = out[:nblk].cpu().double()
    print(json.dumps({"mechanism": names[mode], "chunk": chunk, "stages": stages, "ctas": nblk, "scatter": scatter, "TBps": round(nblk * per / (best * 1e-3) / 1e12, 3),
                      "bytes_per_clk_per_sm_median": round(per / float(cyc.median()), 2)}), flush=True)
for nblk in (nb_max, nb_max // 2):
    for mode, chunk, stages in ((0, 65536, 3), (0, 32768, 6), (0, 16384, 8), (0, 8192, 8), (1, 65536, 3), (1, 32768, 6), (1, 16384, 8),
                                (2, 65536, 2), (2, 65536, 3), (2, 16384, 8), (3, 16384, 1), (4, 16384, 1)):
        run(mode, chunk, stages, nblk)
for mode, chunk, stages in ((0, 65536, 3), (0, 8192, 8), (2, 65536, 3), (2, 16384, 8)):
    run(mode, chunk, stages, nb_max, scatter=1)
