"""What a pure read, a pure write and a copy stream reach on this GPU's HBM -- the ceilings of the training kernels, which are bound by
record writes (training-mode forward, dgrad chain) or record reads (wgrad).  Plain 16-byte loads/stores (libnerf_b200_dev.so) and,
beside them, torch's own fill / copy kernels.  4 GiB buffers (>> the 50 MB L2), best of 5.  Prints one JSON object."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nerf_pytorch_b200 import _lib
dev = torch.device("cuda:0")
lib = _lib.load_dev()
n = 4 << 30
a = torch.empty(n, dtype=torch.uint8, device=dev); b = torch.empty(n, dtype=torch.uint8, device=dev)
a.zero_(); b.zero_()
st = torch.cuda.current_stream().cuda_stream
def t(fn, reps=5):
    fn(); torch.cuda.synchronize()
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best
def probe(mode, blocks):
    return lambda: _lib.check_dev(lib.nerf_b200_debug_hbm_stream(a.data_ptr(), b.data_ptr(), n, mode, blocks, st), "hbm_stream")
res = {"bytes": n}
sms = torch.cuda.get_device_properties(0).multi_processor_count
for blocks in (sms * 2, sms * 4, sms * 8):
    res[f"read_TBps_{blocks}blk"] = n / (t(probe(0, blocks)) * 1e-3) / 1e12
    res[f"write_TBps_{blocks}blk"] = n / (t(probe(1, blocks)) * 1e-3) / 1e12
    res[f"copy_read_plus_write_TBps_{blocks}blk"] = 2 * n / (t(probe(2, blocks)) * 1e-3) / 1e12
res["torch_fill_write_TBps"] = n / (t(lambda: a.zero_()) * 1e-3) / 1e12
res["torch_copy_read_plus_write_TBps"] = 2 * n / (t(lambda: b.copy_(a)) * 1e-3) / 1e12
print(json.dumps(res))
