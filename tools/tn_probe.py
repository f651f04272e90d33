"""MN-major descriptor check for the round-2 weight-gradient GEMM: out = X^T Y through wgmma with both operands
read from activation-layout tiles; sweeps (lbo, sbo) encodings and prints the error of each."""
import ctypes as C, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as ge; ge.build()
from nerf_pytorch_b200 import _lib
lib = _lib.load_dev(); dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
X = torch.randn(128, 256, generator=g); Y = torch.randn(128, 256, generator=g)
ref = (X.half().double().T @ Y.half().double()).numpy()
Xd, Yd = X.to(dev), Y.to(dev)
for lbo, sbo in ((16384, 1024), (1024, 16384), (16384, 128), (128, 16384), (16, 1024), (0, 1024)):
    out = torch.zeros(256, 256, device=dev)
    rc = lib.nerf_b200_selftest_gemm_tn(C.c_void_p(Xd.data_ptr()), C.c_void_p(Yd.data_ptr()), C.c_void_p(out.data_ptr()), lbo, sbo, None)
    torch.cuda.synchronize()
    o = out.cpu().double().numpy()
    err = np.linalg.norm(o - ref) / np.linalg.norm(ref)
    errT = np.linalg.norm(o - ref.T) / np.linalg.norm(ref)
    print(f"lbo={lbo:6d} sbo={sbo:6d} rc={rc}: rel err {err:.3e}  (vs transposed {errT:.3e})  out[0,:4]={o[0,:4]} ref[0,:4]={ref[0,:4]}")
