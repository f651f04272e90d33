"""Shared helpers for the -m gpu parity tests (they call the CUDA library through the C ABI via the
Python host mirror and compare with the numpy oracle / the committed golden fixtures)."""
import ctypes as C

import numpy as np
import torch

import nerf_pytorch_b200 as nb
from nerf_pytorch_b200 import _lib
from nerf_pytorch_b200.api import _QueryFn
from oracle import nerf_oracle as O
from oracle import synth

DEV = torch.device("cuda:0")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def make_net(state, use_viewdirs=True, output_ch=5, D=8, skips=(4,), input_ch=63, input_ch_views=27, W=256):
    m = nb.NeRF(D=D, W=W, input_ch=input_ch, input_ch_views=input_ch_views if use_viewdirs else 0, output_ch=output_ch,
                skips=list(skips), use_viewdirs=use_viewdirs)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    return m.to(DEV)


def query_fn():
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    return _QueryFn(e, ed, 65536, 10, 4, 0)


def packed_rays(fx):
    rays = fx["rays"]
    return O.pack_rays(int(fx["H"]), int(fx["W"]), fx["K"], rays[0], rays[1], bool(fx["ndc"]),
                       float(fx["near"]), float(fx["far"]), True)


def ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- one network pass through the C ABI ---------------------------------------------------------------------------------
# rays [N, 8 | 11] (the packed batch: its width is the ray stride), z [N, S]; L / Lv are multires / multires_views (0 for
# i_embed = -1).

def cfg(S, ray_stride, L=10, Lv=4, white=True, precision=_lib.PREC_TC_FP16):
    c = _lib.NerfRenderCfg()
    c.N_samples, c.N_importance, c.multires, c.multires_views = S, 0, L, Lv
    c.lindisp, c.perturb, c.white_bkgd, c.ray_stride, c.precision = 0, 0, int(white), ray_stride, precision
    return c


def march(net, rays, z, train, L=10, Lv=4, white=True, precision=_lib.PREC_TC_FP16):
    """nerf_b200_march (inference, either precision) or nerf_b200_march_train -> (outputs dict, act, mask); act / mask are
    None when not training.  Outputs: rgb, disp, acc, w (weights), raw."""
    from nerf_pytorch_b200 import api
    lib = _lib.load()
    N, S = z.shape
    n = net.net_params()
    pk = net.packed() if precision == _lib.PREC_TC_FP16 else None
    c = cfg(S, rays.shape[1], L, Lv, white, precision)
    o = {k: torch.zeros(s, device=DEV) for k, s in (("rgb", (N, 3)), ("disp", (N,)), ("acc", (N,)), ("w", (N, S)), ("raw", (N, S, 4)))}
    out = _lib.NerfPassOut(ptr(o["rgb"]), ptr(o["disp"]), ptr(o["acc"]), C.c_void_p(0), ptr(o["w"]), ptr(o["raw"]))
    ws_bytes = max(lib.nerf_b200_march_workspace_bytes(N, S), N * S * 28)     # the exact mode keeps pts and raw there
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    if train:
        sv, act, mask = api._train_save(lib, N, S, n, DEV)
        act.zero_(); mask.zero_()
        _lib.check(lib.nerf_b200_march_train(ptr(rays), ptr(z), None, N, S, C.byref(n), ptr(pk), C.byref(c), C.byref(out),
                                             ptr(ws), ws_bytes, C.byref(sv), stream()), "march_train")
    else:
        act = mask = None
        _lib.check(lib.nerf_b200_march(ptr(rays), ptr(z), None, N, S, C.byref(n), ptr(pk), C.byref(c), C.byref(out),
                                       ptr(ws), ws_bytes, stream()), "march")
    torch.cuda.synchronize()
    return o, act, mask


def _seed_args(seeds):
    """g_rgb tensor -> the rgb-only entry point's argument; dict of output gradients -> NerfOutGrads"""
    if isinstance(seeds, dict):
        return False, _lib.NerfOutGrads(**{k: ptr(v) for k, v in seeds.items()})
    return True, seeds


def march_bwd_tc(net, rays, z, raw, act, mask, seeds, L=10, Lv=4, white=True, on_device=False):
    """nerf_b200_march_bwd_tc (seeds: dL/drgb_map [N, 3]) or nerf_b200_march_bwd_tc_outs (seeds: dict output name -> gradient)
    -> (grads dict name -> np, workspace bytes np from its 1 KB-aligned base; on_device: a uint8 tensor on the device)"""
    lib = _lib.load()
    N, S = z.shape
    n = net.net_params()
    c = cfg(S, rays.shape[1], L, Lv, white)
    grads = {k: torch.zeros_like(p, dtype=torch.float32) for k, p in net.named_parameters()}
    gs = net.grad_struct(grads)
    sv = _lib.NerfTrainSave(ptr(act), act.numel(), ptr(mask), mask.numel())
    ws_bytes = lib.nerf_b200_march_bwd_tc_workspace_bytes(N, S, C.byref(n))
    assert ws_bytes > 0
    ws = torch.zeros(ws_bytes + 1024, dtype=torch.uint8, device=DEV)
    base = (ws.data_ptr() + 1023) // 1024 * 1024 - ws.data_ptr()          # the library aligns the same way
    rgb_only, s = _seed_args(seeds)
    args = (ptr(rays), ptr(z), None, N, S, C.byref(n), ptr(net.packed()), C.byref(c), ptr(raw), C.byref(sv))
    tail = (C.byref(gs), ptr(ws), ws_bytes + 1024, stream())
    if rgb_only:
        _lib.check(lib.nerf_b200_march_bwd_tc(*args, ptr(s), *tail), "march_bwd_tc")
    else:
        _lib.check(lib.nerf_b200_march_bwd_tc_outs(*args, C.byref(s), *tail), "march_bwd_tc_outs")
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in grads.items()}, (ws[base:] if on_device else ws.cpu().numpy()[base:])


def run_network_exact(net, pts, viewdirs, S, L=10, Lv=4):
    """nerf_b200_run_network in fp32: pts [N * S, 3], viewdirs [N, 3] or None -> raw [N * S, 4]"""
    lib = _lib.load()
    N = pts.shape[0] // S
    raw = torch.zeros((N * S, 4), device=DEV)
    _lib.check(lib.nerf_b200_run_network(ptr(pts), ptr(viewdirs), N, S, C.byref(net.net_params()), None, L, Lv, _lib.PREC_FP32,
                                         ptr(raw), None, 0, stream()), "run_network")
    torch.cuda.synchronize()
    return raw


def march_bwd_exact(net, rays, z, seeds, L=10, Lv=4, white=True, fill=None):
    """nerf_b200_march_bwd / nerf_b200_march_bwd_outs (fp32 recompute of the pass) -> grads dict name -> np.  fill: byte the
    workspace is set to before the call (None: left as allocated)"""
    lib = _lib.load()
    N, S = z.shape
    n = net.net_params()
    c = cfg(S, rays.shape[1], L, Lv, white, _lib.PREC_FP32)
    grads = {k: torch.zeros_like(p, dtype=torch.float32) for k, p in net.named_parameters()}
    gs = net.grad_struct(grads)
    ws_bytes = lib.nerf_b200_march_bwd_workspace_bytes(N, S, C.byref(n))
    assert ws_bytes > 0
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    if fill is not None:
        ws.fill_(fill)
    rgb_only, s = _seed_args(seeds)
    args = (ptr(rays), ptr(z), None, N, S, C.byref(n), None, C.byref(c))
    tail = (C.byref(gs), ptr(ws), ws_bytes, stream())
    if rgb_only:
        _lib.check(lib.nerf_b200_march_bwd(*args, ptr(s), *tail), "march_bwd")
    else:
        _lib.check(lib.nerf_b200_march_bwd_outs(*args, C.byref(s), *tail), "march_bwd_outs")
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in grads.items()}
