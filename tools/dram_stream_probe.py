"""Per-SM HBM streaming rates of the copy mechanisms the training kernels can use (libnerf_b200_dev.so: dram_stream_probe_kernel):
cp.async.bulk global->shared rings, 16-byte cp.async rings, cp.async.bulk shared->global, plain vector loads / stores.
One CTA per SM, disjoint 16 MiB regions per CTA and launch (8 launches walk a 19 GB buffer: nothing is re-read from L2).
Prints JSON lines: mechanism, ring, CTAs, TB/s (CUDA events) and bytes/clock/SM (clock64 inside the kernel, median CTA).

--l2: instead, the L2 -> SM ceiling of the fused forward's weight stream: every CTA streams the SAME 1 179 648 bytes (the
forward's chunk sequence at D = 8 with view directions: 68 x 16 KB + 8 x 8 KB) through a cp.async.bulk ring of 16 KB stages,
as march_wg_kernel's producer does, at 128 CTAs (the bench shape's tile plan) and one per SM."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nerf_pytorch_b200 import _lib
dev = torch.device("cuda:0")
lib = _lib.load_dev()
per = 16 << 20
nb_max = torch.cuda.get_device_properties(0).multi_processor_count
if "--l2" in sys.argv:
    FWD_CHUNK_BYTES = 68 * 16384 + 8 * 8192
    region = torch.randint(0, 256, (FWD_CHUNK_BYTES,), dtype=torch.uint8, device=dev)
    out = torch.zeros(nb_max + 8, dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    total = 64 * FWD_CHUNK_BYTES                        # bytes per CTA and launch: the sequence 64 times
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}), flush=True)
    for nblk in (128, nb_max):
        for stages in (6, 7, 8):
            best, cyc = 1e9, None
            for rep in range(6):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _lib.check_dev(lib.nerf_b200_debug_l2_stream(region.data_ptr(), total, FWD_CHUNK_BYTES, 16384, stages, 0, nblk, 0,
                                                             out.data_ptr(), st), "l2_stream")
                e1.record(); torch.cuda.synchronize()
                if rep >= 1 and e0.elapsed_time(e1) < best:
                    best = e0.elapsed_time(e1); cyc = out[:nblk].cpu().double()
            print(json.dumps({"mechanism": "cp.async.bulk g2s, L2-resident shared region", "region_bytes": FWD_CHUNK_BYTES, "chunk": 16384,
                              "stages": stages, "ctas": nblk, "TBps": round(nblk * total / (best * 1e-3) / 1e12, 3),
                              "bytes_per_clk_per_sm_median": round(total / float(cyc.median()), 2)}), flush=True)
    sys.exit(0)
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
