"""Host-side mirror of the reference's renderer interface (run_nerf.py / run_nerf_helpers.py).

Same names, argument meaning and return structure as yenchenlin/nerf-pytorch, so that these
functions can be rebound onto the reference's `run_nerf` module (see dropin.py) and `train()`
runs unchanged -- but every tensor-op chain of the hot path is one call into the hand-written
sm_90a library behind include/nerf_b200.h.  PyTorch is used for memory, streams and autograd
plumbing only.  There is no CPU fallback: tensors must live on a CUDA device.

Reference sites: render run_nerf.py:69-134, batchify_rays :54-66, render_rays :308-418,
run_network :37-51, batchify :27-34, raw2outputs :262-305, create_nerf :178-259;
Embedder/get_embedder run_nerf_helpers.py:15-63, NeRF :67-119, get_rays :153-162,
ndc_rays :175-192, sample_pdf :196-239.
"""
from __future__ import annotations

import ctypes as C
import numbers
import os
from typing import NamedTuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from ._lib import (NerfCamera, NerfNetGrads, NerfNetParams, NerfPassOut, NerfRenderCfg, NerfTrainSave, PREC_FP32, PREC_TC_FP16,
                   PREC_TC_SPLIT, check)

__all__ = ["NeRF", "Embedder", "get_embedder", "sample_pdf", "raw2outputs", "run_network", "batchify",
           "batchify_rays", "render_rays", "render", "create_nerf",
           "img2mse", "mse2psnr", "to8b", "set_precision", "get_precision", "set_backward", "get_backward",
           "launch_count", "DEBUG", "GraphedRender", "render_to8b", "DeviceRayBatcher", "density_grid", "marching_cubes",
           "extract_mesh", "save_ply", "density_gradient", "vertex_attributes"]

DEBUG = False
_PRECISION = {"mode": PREC_TC_FP16}

img2mse = lambda x, y: torch.mean((x - y) ** 2)                                    # run_nerf_helpers.py:9
mse2psnr = lambda x: -10. * torch.log(x) / torch.log(torch.tensor([10.], device=x.device))   # :10
to8b = lambda x: (255 * np.clip(x, 0, 1)).astype(np.uint8)                          # :11


_PRECISIONS = {"tc_fp16": PREC_TC_FP16, "fp32": PREC_FP32, "tc_split": PREC_TC_SPLIT}


def set_precision(mode: str):
    """'tc_fp16' (wgmma fp16 operands / fp32 accumulate, default), 'fp32' (CUDA-core exact mode) or 'tc_split' (wgmma with
    every operand split into hi + lo fp16 halves, three MMAs per K-step into an fp32 accumulator: the fp32 path's accuracy on
    tensor cores, for the forward; netwidth 256 only, like tc_fp16)."""
    _PRECISION["mode"] = _PRECISIONS[mode]


def get_precision() -> str:
    return {v: k for k, v in _PRECISIONS.items()}[_PRECISION["mode"]]


def set_backward(mode: str):
    """'tc' (default in tc_fp16 precision: wgmma backward from the forward's saved tile records, with or without view
    directions), 'exact' (fp32 CUDA-core recompute backward; always used in fp32 precision, and in tc_split precision unless
    'tc_split' is selected: the split tensor-core forward, then the pass recomputed in fp32 on CUDA cores) or 'tc_split'
    (precision tc_split only: the split training forward leaves hi + lo tile records and the backward runs on tensor cores
    with every operand split into hi + lo fp16 halves; a call that needs gradients in another precision raises)."""
    if mode not in ("tc", "exact", "tc_split"):
        raise ValueError(mode)
    _PRECISION["backward"] = mode


def get_backward() -> str:
    return _PRECISION.get("backward", "tc")


def launch_count() -> int:
    return _lib.launch_count()


# ------------------------------------------------------------------------------------------------
# small helpers
# ------------------------------------------------------------------------------------------------

def _stream(t: torch.Tensor):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _on(t: torch.Tensor):
    """Make the tensor's device the current CUDA device for the duration of a library call: the C library launches
    on the process's current device (per-device state lives in csrc/capi.cu: device_state())."""
    return torch.cuda.device(t.device)


def _ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _call(lib, name, *args):
    """Call the library entry `name` and raise its error under the name without the nerf_b200_ prefix.  Callers spell `name`
    out in full, so that a search for an entry point finds them."""
    check(getattr(lib, name)(*args), name[len("nerf_b200_"):])


def _f32c(t: torch.Tensor, what: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"nerf_b200: {what} must be a CUDA tensor (no CPU fallback exists)")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


# ------------------------------------------------------------------------------------------------
# Embedder  (run_nerf_helpers.py:15-63)
# ------------------------------------------------------------------------------------------------

class Embedder:
    """Positional encoding [x, sin(2^k x), cos(2^k x)]_{k<L}; same kwargs as the reference's
    Embedder, restricted to what get_embedder ever passes (include_input, log_sampling, sin/cos)."""

    def __init__(self, **kwargs):
        self.kwargs = kwargs
        if not (kwargs.get("include_input", True) and kwargs.get("log_sampling", True) and kwargs.get("input_dims", 3) == 3):
            raise NotImplementedError("nerf_b200 Embedder supports include_input=True, log_sampling=True, input_dims=3")
        self.num_freqs = int(kwargs["num_freqs"])
        if int(kwargs.get("max_freq_log2", self.num_freqs - 1)) != self.num_freqs - 1:
            raise NotImplementedError("nerf_b200 Embedder needs max_freq_log2 == num_freqs - 1 (powers of two)")
        self.out_dim = 3 + 6 * self.num_freqs

    def embed(self, inputs: torch.Tensor) -> torch.Tensor:
        x = _f32c(inputs, "embed input")
        flat = x.reshape(-1, 3)
        out = torch.empty((flat.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        with _on(x):
            check(_lib.load().nerf_b200_embed(_ptr(flat), flat.shape[0], self.num_freqs, _ptr(out), _stream(x)), "embed")
        return out.reshape(*x.shape[:-1], self.out_dim)


def get_embedder(multires, i=0):
    """run_nerf_helpers.py:48-63."""
    if i == -1:
        return nn.Identity(), 3
    eo = Embedder(include_input=True, input_dims=3, max_freq_log2=multires - 1, num_freqs=multires,
                  log_sampling=True, periodic_fns=[torch.sin, torch.cos])
    embed = lambda x, eo=eo: eo.embed(x)
    embed.num_freqs = multires          # lets run_network recover L without re-deriving it
    return embed, eo.out_dim


# ------------------------------------------------------------------------------------------------
# NeRF module  (run_nerf_helpers.py:67-119): parameter container with the reference's state_dict keys
# ------------------------------------------------------------------------------------------------

def effective_skip(skips, D):
    """The one skip connection of a D-layer net (-1: none).  The reference's forward concatenates after layer i only for
    i in range(D) (run_nerf_helpers.py:99-103), so entries >= D and negative ones never take effect: create_nerf's
    skips = [4] with netdepth <= 4 is a net without a skip.  Entry D - 1 stays and is rejected by the library, as the
    reference fails on it (its heads would receive W + input_ch columns)."""
    live = [s for s in skips if 0 <= s < D]
    if len(live) > 1:
        raise NotImplementedError("nerf_b200 supports at most one skip connection")
    return live[0] if live else -1


class NeRF(nn.Module):
    def __init__(self, D=8, W=256, input_ch=3, input_ch_views=3, output_ch=4, skips=[4], use_viewdirs=False):
        super().__init__()
        self.D, self.W = D, W
        self.input_ch, self.input_ch_views = input_ch, input_ch_views
        self.skips, self.use_viewdirs, self.output_ch = skips, use_viewdirs, output_ch
        self.pts_linears = nn.ModuleList(
            [nn.Linear(input_ch, W)] + [nn.Linear(W, W) if i not in self.skips else nn.Linear(W + input_ch, W)
                                        for i in range(D - 1)])
        self.views_linears = nn.ModuleList([nn.Linear(input_ch_views + W, W // 2)])
        if use_viewdirs:
            self.feature_linear = nn.Linear(W, W)
            self.alpha_linear = nn.Linear(W, 1)
            self.rgb_linear = nn.Linear(W // 2, 3)
        else:
            self.output_linear = nn.Linear(W, output_ch)
        self._pack = None           # (key, packed fp16 weight stream) for the tensor-core path
        self._pack_split = None     # (key, split hi | lo image) for precision tc_split

    def forward(self, x):
        """Evaluate on ALREADY-EMBEDDED rows [M, input_ch + input_ch_views] (run_nerf_helpers.py:96-119).

        Interface parity only: the renderer never calls this (the fused kernel encodes and evaluates
        the MLP itself from ray / sample coordinates); it exists so user code that calls
        `network_fn(embedded)` keeps working, and uses plain torch ops."""
        input_pts, input_views = torch.split(x, [self.input_ch, self.input_ch_views], dim=-1)
        h = input_pts
        for i, l in enumerate(self.pts_linears):
            h = F.relu(l(h))
            if i in self.skips:
                h = torch.cat([input_pts, h], -1)
        if self.use_viewdirs:
            alpha = self.alpha_linear(h)
            feature = self.feature_linear(h)
            h = torch.cat([feature, input_views], -1)
            for l in self.views_linears:
                h = F.relu(l(h))
            return torch.cat([self.rgb_linear(h), alpha], -1)
        return self.output_linear(h)

    # ---- C-ABI views of the live parameter storages ------------------------------------------
    def _named_params(self):
        """list(self.named_parameters()), cached: walking the module tree costs ~50 us per network and every render_rays call needs
        the list several times.  The cache holds (owner module, attribute, name, parameter) and is valid as long as every owner
        still holds that very Parameter object (assigning a new Parameter to a layer rebuilds it)."""
        c = self.__dict__.get("_np_cache")
        if c is not None and all(m._parameters.get(a) is q for m, a, _, q in c):
            return c
        c = []
        for name, q in self.named_parameters():
            prefix, _, attr = name.rpartition(".")
            c.append((self.get_submodule(prefix) if prefix else self, attr, name, q))
        self.__dict__["_np_cache"] = c
        return c

    def _check_device(self):
        p = self.pts_linears[0].weight
        if not p.is_cuda:
            raise RuntimeError("nerf_b200: NeRF parameters must be on a CUDA device (no CPU fallback exists)")
        return p.device

    def net_params(self) -> NerfNetParams:
        if not 1 <= self.D <= _lib.MAX_D:
            raise RuntimeError(f"nerf_b200: netdepth must be in [1, {_lib.MAX_D}] (got {self.D})")
        self._check_device()
        n = NerfNetParams()
        n.D, n.W, n.input_ch = self.D, self.W, self.input_ch
        n.input_ch_views = self.input_ch_views if self.use_viewdirs else 0
        n.skip = effective_skip(self.skips, self.D)
        n.use_viewdirs, n.output_ch = int(self.use_viewdirs), self.output_ch
        for i, l in enumerate(self.pts_linears):
            if not (l.weight.is_contiguous() and l.weight.dtype == torch.float32):
                raise RuntimeError("nerf_b200: parameters must be contiguous fp32")
            n.pts_w[i], n.pts_b[i] = l.weight.data_ptr(), l.bias.data_ptr()
        if self.use_viewdirs:
            n.feature_w, n.feature_b = self.feature_linear.weight.data_ptr(), self.feature_linear.bias.data_ptr()
            n.alpha_w, n.alpha_b = self.alpha_linear.weight.data_ptr(), self.alpha_linear.bias.data_ptr()
            n.views_w, n.views_b = self.views_linears[0].weight.data_ptr(), self.views_linears[0].bias.data_ptr()
            n.rgb_w, n.rgb_b = self.rgb_linear.weight.data_ptr(), self.rgb_linear.bias.data_ptr()
        else:
            n.output_w, n.output_b = self.output_linear.weight.data_ptr(), self.output_linear.bias.data_ptr()
        return n

    def grad_struct(self, grads: dict) -> NerfNetGrads:
        """grads: name -> fp32 CUDA tensor shaped like the parameter (see named_parameters())."""
        g = NerfNetGrads()
        for i in range(self.D):
            g.pts_w[i], g.pts_b[i] = grads[f"pts_linears.{i}.weight"].data_ptr(), grads[f"pts_linears.{i}.bias"].data_ptr()
        if self.use_viewdirs:
            for nm in ("feature", "alpha", "rgb"):
                setattr(g, nm + "_w", grads[f"{nm}_linear.weight"].data_ptr())
                setattr(g, nm + "_b", grads[f"{nm}_linear.bias"].data_ptr())
            g.views_w, g.views_b = grads["views_linears.0.weight"].data_ptr(), grads["views_linears.0.bias"].data_ptr()
        else:
            g.output_w, g.output_b = grads["output_linear.weight"].data_ptr(), grads["output_linear.bias"].data_ptr()
        return g

    def load_weights_from_keras(self, weights):
        """Import the original TF/Keras NeRF's weight list (same contract as run_nerf_helpers.py:121-148): kernels arrive as
        [in, out] arrays in the order pts_linears (D), feature, views, rgb, alpha, each followed by its bias.  The layers
        keep their Parameters (copy_ under no_grad, on whatever device they live), so the optimizer and the packed
        tensor-core copy stay valid; the reference re-binds `.data` to CPU tensors instead."""
        if not self.use_viewdirs:
            raise AssertionError("Not implemented if use_viewdirs=False")
        order = list(self.pts_linears) + [self.feature_linear, self.views_linears[0], self.rgb_linear, self.alpha_linear]
        with torch.no_grad():
            for i, lin in enumerate(order):
                lin.weight.copy_(torch.as_tensor(np.ascontiguousarray(np.asarray(weights[2 * i]).T), dtype=lin.weight.dtype))
                lin.bias.copy_(torch.as_tensor(np.asarray(weights[2 * i + 1]).reshape(-1), dtype=lin.bias.dtype))
        self.invalidate_pack()

    def invalidate_pack(self):
        """Force the next packed() to re-pack.  Needed after writes that autograd's version counter does not see
        (`p.data.copy_()`, `p.data.mul_()` -- e.g. EMA or clipping through `.data`); optimizer steps, `copy_` under
        no_grad, load_state_dict and .to() are detected automatically."""
        self._pack_epoch = getattr(self, "_pack_epoch", 0) + 1

    def packed(self):
        """fp16 UMMA-swizzled weight streams (forward chunks + the transposed chunks of the backward), re-packed
        whenever a parameter changed in place (optimizer.step bumps Parameter._version; load_state_dict / .to()
        change data_ptr) or invalidate_pack() was called."""
        return self._packed_image("_pack", "nerf_b200_packed_bytes", "nerf_b200_pack_weights")

    def packed_split(self):
        """The split image of precision tc_split (hi | lo fp16 halves of the scaled forward weights), cached apart from
        packed() and re-packed on the same conditions."""
        return self._packed_image("_pack_split", "nerf_b200_packed_bytes_split", "nerf_b200_pack_weights_split")

    def packed_split_train(self):
        """The split training image of set_backward('tc_split'): packed_split()'s bytes followed by the backward's transposed
        chunks as hi | lo halves, cached apart from the other images and re-packed on the same conditions."""
        return self._packed_image("_pack_split_train", "nerf_b200_packed_bytes_split_train", "nerf_b200_pack_weights_split_train")

    def _packed_image(self, attr, size_fn, pack_fn):
        dev = self._check_device()
        key = (getattr(self, "_pack_epoch", 0),) + tuple((q.data_ptr(), q._version) for _, _, _, q in self._named_params())
        cached = getattr(self, attr, None)
        if cached is not None and cached[0] == key:
            return cached[1]
        lib = _lib.load()
        n = self.net_params()
        nbytes = getattr(lib, size_fn)(C.byref(n))
        if nbytes == 0:
            raise RuntimeError("nerf_b200: " + lib.nerf_b200_last_error().decode())
        buf = cached[1] if (cached is not None and cached[1].numel() == nbytes and cached[1].device == dev) \
            else torch.empty(nbytes, dtype=torch.uint8, device=dev)
        with _on(buf):
            _call(lib, pack_fn, C.byref(n), _ptr(buf), nbytes, _stream(buf))
        setattr(self, attr, (key, buf))
        return buf


# ------------------------------------------------------------------------------------------------
# sample_pdf  (run_nerf_helpers.py:196-239)
# ------------------------------------------------------------------------------------------------

def _draw_u(shape, det, pytest, device):
    """The `u` of sample_pdf (run_nerf_helpers.py:204-219) -> (tensor, row_stride)."""
    n_rows, n = shape
    if pytest:
        np.random.seed(0)
        if det:
            return torch.tensor(np.linspace(0., 1., n), dtype=torch.float32, device=device), 0
        return torch.tensor(np.random.rand(n_rows, n), dtype=torch.float32, device=device), n
    if det:
        return torch.linspace(0., 1., steps=n, device=device), 0
    return torch.rand(n_rows, n, device=device), n


def sample_pdf(bins, weights, N_samples, det=False, pytest=False):
    bins, weights = _f32c(bins, "bins"), _f32c(weights, "weights")
    lead = bins.shape[:-1]
    B = bins.shape[-1]
    b2, w2 = bins.reshape(-1, B), weights.reshape(-1, B - 1)
    u, stride = _draw_u((b2.shape[0], N_samples), det, pytest, bins.device)
    out = torch.empty((b2.shape[0], N_samples), device=bins.device, dtype=torch.float32)
    with _on(bins):
        check(_lib.load().nerf_b200_sample_pdf(_ptr(b2), _ptr(w2), _ptr(u), stride, b2.shape[0], B, N_samples,
                                               _ptr(out), _stream(bins)), "sample_pdf")
    return out.reshape(*lead, N_samples)


# ------------------------------------------------------------------------------------------------
# raw2outputs  (run_nerf.py:262-305), differentiable w.r.t. raw through rgb_map
# ------------------------------------------------------------------------------------------------

def _draw_noise(shape, std, pytest, device):
    """sigma noise of raw2outputs (run_nerf.py:283-291); note the pytest path is uniform, the live path normal."""
    if std > 0.:
        if pytest:
            np.random.seed(0)
            return torch.tensor(np.random.rand(*shape) * std, dtype=torch.float32, device=device)
        return torch.randn(shape, device=device) * std
    return None


class _Raw2Outputs(torch.autograd.Function):
    @staticmethod
    def forward(ctx, raw, z_vals, rays_d, noise, white_bkgd):
        N, S = z_vals.shape
        dev = raw.device
        rgb = torch.empty((N, 3), device=dev); disp = torch.empty(N, device=dev); acc = torch.empty(N, device=dev)
        depth = torch.empty(N, device=dev); weights = torch.empty((N, S), device=dev)
        out = NerfPassOut(_ptr(rgb), _ptr(disp), _ptr(acc), _ptr(depth), _ptr(weights), C.c_void_p(0))
        with _on(raw):
            check(_lib.load().nerf_b200_raw2outputs(_ptr(raw), _ptr(z_vals), _ptr(rays_d), 3, _ptr(noise), N, S,
                                                    int(white_bkgd), C.byref(out), _stream(raw)), "raw2outputs")
        ctx.save_for_backward(raw, z_vals, rays_d, noise if noise is not None else torch.empty(0, device=dev))
        ctx.white_bkgd = bool(white_bkgd)
        ctx.set_materialize_grads(False)
        return rgb, disp, acc, weights, depth

    @staticmethod
    def backward(ctx, g_rgb, g_disp, g_acc, g_weights, g_depth):
        raw, z_vals, rays_d, noise = ctx.saved_tensors
        noise = noise if noise.numel() else None
        N, S = z_vals.shape
        d_raw = torch.empty_like(raw)
        lib = _lib.load()
        args = (_ptr(raw), _ptr(z_vals), _ptr(rays_d), 3, _ptr(noise), N, S, int(ctx.white_bkgd))
        with _on(raw):
            if g_disp is None and g_acc is None and g_weights is None and g_depth is None:
                g_rgb = g_rgb.contiguous().float()
                check(lib.nerf_b200_raw2outputs_bwd(*args, _ptr(g_rgb), _ptr(d_raw), _stream(raw)), "raw2outputs_bwd")
            else:
                og, keep = _out_grads(rgb_map=g_rgb, disp_map=g_disp, acc_map=g_acc, depth_map=g_depth, weights=g_weights)
                check(lib.nerf_b200_raw2outputs_bwd_outs(*args, C.byref(og), _ptr(d_raw), _stream(raw)), "raw2outputs_bwd_outs")
        return d_raw, None, None, None, None


def _out_grads(**seeds):
    """NerfOutGrads over the given output gradients (None -> NULL) -> (struct, the contiguous fp32 tensors it points to)."""
    keep = {k: v.contiguous().float() for k, v in seeds.items() if v is not None}
    return _lib.NerfOutGrads(**{k: _ptr(v) for k, v in keep.items()}), keep


def raw2outputs(raw, z_vals, rays_d, raw_noise_std=0, white_bkgd=False, pytest=False):
    """-> rgb_map, disp_map, acc_map, weights, depth_map, all differentiable w.r.t. `raw` as in the reference
    (nerf_b200_raw2outputs_bwd_outs; a loss on rgb_map alone takes nerf_b200_raw2outputs_bwd)."""
    raw, z_vals, rays_d = _f32c(raw, "raw"), _f32c(z_vals, "z_vals"), _f32c(rays_d, "rays_d")
    if raw.shape[-1] != 4:
        raw = raw[..., :4].contiguous()
    noise = _draw_noise(tuple(z_vals.shape), float(raw_noise_std), pytest, raw.device)
    return _Raw2Outputs.apply(raw, z_vals, rays_d, noise, white_bkgd)


# ------------------------------------------------------------------------------------------------
# run_network / batchify  (run_nerf.py:27-51)
# ------------------------------------------------------------------------------------------------

def batchify(fn, chunk):
    """run_nerf.py:27-34 (kept for interface parity; the fused path needs no chunking)."""
    if chunk is None:
        return fn
    def ret(inputs):
        return torch.cat([fn(inputs[i:i + chunk]) for i in range(0, inputs.shape[0], chunk)], 0)
    return ret


def _freqs_of(embed_fn, out_dim_hint=None):
    if embed_fn is None:
        return 0
    if isinstance(embed_fn, nn.Identity):
        return 0
    L = getattr(embed_fn, "num_freqs", None)
    if L is None:
        raise RuntimeError("nerf_b200.run_network needs embedders created by nerf_b200.get_embedder")
    return int(L)


def _packed_for(net, prec):
    """The packed image a precision reads: packed() for tc_fp16, packed_split() for tc_split, None for fp32."""
    if prec == PREC_TC_FP16:
        return net.packed()
    return net.packed_split() if prec == PREC_TC_SPLIT else None


def run_network(inputs, viewdirs, fn, embed_fn, embeddirs_fn, netchunk=1024 * 64):
    """inputs [N,S,3] (+ viewdirs [N,3]) -> raw [N,S,4] in ONE fused kernel: encode + MLP.
    `netchunk` is accepted and ignored ("does not affect final results", run_nerf.py:78-79)."""
    if not isinstance(fn, NeRF):
        raise RuntimeError("nerf_b200.run_network: network must be a nerf_b200.NeRF")
    inputs = _f32c(inputs, "inputs")
    N, S = int(np.prod(inputs.shape[:-2])) if inputs.dim() > 2 else 1, inputs.shape[-2]
    pts = inputs.reshape(-1, 3)
    vd = _f32c(viewdirs, "viewdirs").reshape(-1, 3) if viewdirs is not None else None
    lib = _lib.load()
    n = fn.net_params()
    prec = _PRECISION["mode"]
    packed = _packed_for(fn, prec)
    raw = torch.empty((N * S, 4), device=inputs.device, dtype=torch.float32)
    ws_bytes = lib.nerf_b200_march_workspace_bytes(N, S)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=inputs.device)
    with _on(inputs):
        check(lib.nerf_b200_run_network(_ptr(pts), _ptr(vd), N, S, C.byref(n), _ptr(packed), _freqs_of(embed_fn),
                                        _freqs_of(embeddirs_fn), prec, _ptr(raw), _ptr(ws), ws_bytes, _stream(inputs)),
              "run_network")
    return raw.reshape(*inputs.shape[:-1], 4)


# ------------------------------------------------------------------------------------------------
# render_rays  (run_nerf.py:308-418)
# ------------------------------------------------------------------------------------------------

class _QueryFn:
    """The `network_query_fn` closure of create_nerf (run_nerf.py:201-204) as an object, so that
    render_rays can read the encoder settings instead of calling back into Python per chunk."""

    def __init__(self, embed_fn, embeddirs_fn, netchunk, multires, multires_views, i_embed):
        self.embed_fn, self.embeddirs_fn, self.netchunk = embed_fn, embeddirs_fn, netchunk
        self.multires = 0 if i_embed == -1 else multires
        self.multires_views = 0 if i_embed == -1 else multires_views

    def __call__(self, inputs, viewdirs, network_fn):
        return run_network(inputs, viewdirs, network_fn, self.embed_fn, self.embeddirs_fn, self.netchunk)


def _grad_buffers(net: NeRF):
    """Zeroed fp32 gradient tensors shaped like the parameters: views of ONE flat buffer (one memset instead of 24 fills)."""
    named = list(net.named_parameters())
    flat = torch.zeros(sum(p.numel() for _, p in named), dtype=torch.float32, device=named[0][1].device)
    out, off = {}, 0
    for k, p in named:
        out[k] = flat[off:off + p.numel()].view_as(p)
        off += p.numel()
    return out


_LINSPACE = {}


def _linspace01(n, dev):
    """torch.linspace(0, 1, n) on `dev`, cached (the reference rebuilds it on every call)."""
    key = (n, str(dev))
    t = _LINSPACE.get(key)
    if t is None:
        t = _LINSPACE[key] = torch.linspace(0., 1., steps=n, device=dev)
    return t


def _cfg_struct(cfgd, ray_stride):
    cfg = NerfRenderCfg()
    cfg.N_samples, cfg.N_importance = cfgd["N_samples"], cfgd["N_importance"]
    cfg.multires, cfg.multires_views = cfgd["multires"], cfgd["multires_views"]
    cfg.lindisp, cfg.perturb, cfg.white_bkgd = int(cfgd["lindisp"]), int(cfgd["perturb"] > 0.), int(cfgd["white_bkgd"])
    cfg.ray_stride, cfg.precision = ray_stride, _PRECISION["mode"]
    return cfg


class _TcTrain(NamedTuple):
    """One tensor-core training path: what differs between the fp16 and the split path.  `image` is the NeRF method giving the
    packed image the path reads, `packed_bytes` / `pack_weights` size and pack it into a buffer of the caller's (FusedTrainStep).
    The backward of one pass (`march_bwd*`) or of both passes in one call (`bwd*`) takes NerfOutGrads seeds; the `_rgb` entries
    take dL/drgb_map alone (in NerfBwdPass.g_rgb for `bwd_rgb`) and are None where the path has no such entry."""
    image: object
    packed_bytes: str
    pack_weights: str
    record_bytes: str
    fwd: str
    march_bwd_rgb: str | None
    march_bwd: str
    march_bwd_ws: str
    bwd_rgb: str | None
    bwd: str
    bwd_ws: str


_TC_FP16 = _TcTrain(image=NeRF.packed, packed_bytes="nerf_b200_packed_bytes", pack_weights="nerf_b200_pack_weights",
                    record_bytes="nerf_b200_train_record_bytes", fwd="nerf_b200_render_rays_fwd_train",
                    march_bwd_rgb="nerf_b200_march_bwd_tc", march_bwd="nerf_b200_march_bwd_tc_outs",
                    march_bwd_ws="nerf_b200_march_bwd_tc_workspace_bytes", bwd_rgb="nerf_b200_render_rays_bwd_tc",
                    bwd="nerf_b200_render_rays_bwd_tc_outs", bwd_ws="nerf_b200_render_rays_bwd_tc_workspace_bytes")
_TC_SPLIT = _TcTrain(image=NeRF.packed_split_train, packed_bytes="nerf_b200_packed_bytes_split_train",
                     pack_weights="nerf_b200_pack_weights_split_train", record_bytes="nerf_b200_train_record_bytes_split",
                     fwd="nerf_b200_render_rays_fwd_train_split", march_bwd_rgb=None, march_bwd="nerf_b200_march_bwd_split",
                     march_bwd_ws="nerf_b200_march_bwd_split_workspace_bytes", bwd_rgb=None, bwd="nerf_b200_render_rays_bwd_split",
                     bwd_ws="nerf_b200_render_rays_bwd_split_workspace_bytes")


def _train_path(precision, backward, want_grad, net_c=None, net_f=None, fused=False):
    """The backward a call takes, from get_precision(), get_backward(), whether it needs gradients and its coarse and fine
    networks (net_f None: no fine pass) -> None (no gradient needed), "exact" (the fp32 recompute backward) or the
    tensor-core path whose training forward leaves the records its backward reads (_TC_FP16, _TC_SPLIT).  Raises the refusals.

    A drop-in call (render, render_rays) trains on fp16 records under tc_fp16 with set_backward('tc'), but takes the exact
    backward when its networks disagree on use_viewdirs; set_backward('tc_split') trains on split records under tc_split only.
    FusedTrainStep (fused=True) always trains on records: under tc_fp16 on the fp16 path whatever set_backward says, under
    tc_split with set_backward('tc_split'), and with networks that agree on use_viewdirs (they share the ray batch)."""
    if not want_grad:
        return None
    fp16 = precision == "tc_fp16" and (backward == "tc" or fused)
    split = precision == "tc_split" and backward == "tc_split"
    if fused and not (fp16 or split):
        raise RuntimeError("FusedTrainStep runs the tensor-core path (set_precision('tc_fp16'), or set_precision('tc_split') with "
                           "set_backward('tc_split'))")
    if backward == "tc_split" and not split and not fused:
        raise RuntimeError(f"set_backward('tc_split') needs precision tc_split (precision is {precision}): "
                           "call set_precision('tc_split') or set_backward('tc')")
    if net_f is not None and bool(net_f.use_viewdirs) != bool(net_c.use_viewdirs):
        if fused:
            raise RuntimeError("FusedTrainStep: coarse and fine networks must agree on use_viewdirs (they share the ray batch)")
        if split:
            raise RuntimeError("set_backward('tc_split') needs the coarse and fine networks to agree on use_viewdirs")
        return "exact"
    return _TC_FP16 if fp16 else _TC_SPLIT if split else "exact"


def _record_bytes(lib, path, N, S, net_params):
    """(activation bytes, mask bytes) of the per-tile records one training-mode pass of `path` leaves (csrc/train_common.cuh)."""
    ab, mb = C.c_size_t(0), C.c_size_t(0)
    _call(lib, path.record_bytes, N, S, C.byref(net_params), C.byref(ab), C.byref(mb))
    return ab.value, mb.value


def _train_save(lib, N, S, net_params, dev, path=_TC_FP16):
    """Allocate the records of one training-mode pass of `path` -> (NerfTrainSave, act, mask)."""
    ab, mb = _record_bytes(lib, path, N, S, net_params)
    act = torch.empty(ab, dtype=torch.uint8, device=dev)
    mask = torch.empty(mb, dtype=torch.uint8, device=dev)
    return _records_save(act, mask), act, mask


def _records_save(act, mask):
    """NerfTrainSave over the records (uint8 tensors) of one training-mode pass."""
    return NerfTrainSave(_ptr(act), act.numel(), _ptr(mask), mask.numel())


def _bwd_pass(z, noise, S, net_params, packed, raw, save, g_rgb, grads):
    """NerfBwdPass of one tensor-core backward pass (it keeps the structs it points to alive)."""
    return _lib.NerfBwdPass(_ptr(z), _ptr(noise), S, C.pointer(net_params), _ptr(packed), _ptr(raw), C.pointer(save), _ptr(g_rgb),
                            C.pointer(grads))


def _workspace(nbytes, dev):
    return torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)


# render() -> batchify_rays -> render_rays -> _RenderRays.forward: when the whole image is ONE chunk, render() does not launch
# nerf_b200_pack_rays itself but leaves (batch tensor, NerfRayGen + the objects it points to) here; the forward of that very
# tensor hands the generator to nerf_b200_render_fwd, whose per-ray prologue launch builds the batch (4 launches per step
# instead of 5).  Anything else that touches the batch first must call _flush_deferred_pack().
_DEFERRED_PACK = None


def _launch_pack(lib, gen, out):
    g = gen[0]
    check(lib.nerf_b200_pack_rays(g.rays_o, g.rays_d, g.view_src, g.cam, out.shape[0], g.pixel0, g.ndc, g.near, g.far, g.use_viewdirs,
                                  _ptr(out), _stream(out)), "pack_rays")


def _take_deferred_pack(ray_batch):
    global _DEFERRED_PACK
    d = _DEFERRED_PACK
    if d is None:
        return None
    _DEFERRED_PACK = None
    if d[0].data_ptr() == ray_batch.data_ptr() and d[0].shape == ray_batch.shape:
        return d[1]
    with _on(d[0]):                                          # a different tensor reached the forward: build the batch the plain way
        _launch_pack(_lib.load(), d[1], d[0])
    return None


def _flush_deferred_pack():
    global _DEFERRED_PACK
    d = _DEFERRED_PACK
    if d is not None:
        _DEFERRED_PACK = None
        with _on(d[0]):
            _launch_pack(_lib.load(), d[1], d[0])


class _RenderRays(torch.autograd.Function):
    """Forward: nerf_b200_render_rays_fwd (coarse z -> fused pass -> resample -> fused pass); on a tensor-core training path
    (_train_path) that path's training-mode variant, which also leaves the per-tile activation records.  Backward: per pass
    the path's dgrad chain + layer-major wgrad from those records, or on the exact path nerf_b200_march_bwd (fp32 recompute +
    GEMM backprop).  Every output but z_std carries a gradient, as in the reference: a loss on rgb_map / rgb0 alone
    (run_nerf.py:765-772) takes the rgb-only entry points where the path has them, a loss that also reads disp, acc, disp0,
    acc0 or raw takes their _outs variants (NerfOutGrads seeds per pass).  z_samples is detached in the reference (:394) so
    nothing flows through the resampling."""

    @staticmethod
    def forward(ctx, ray_batch, cfgd, path, net_c, net_f, t_rand, u_rand, noise0, noise1, *params):
        lib = _lib.load()
        dev = ray_batch.device
        N = ray_batch.shape[0]
        Sc, Ni = cfgd["N_samples"], cfgd["N_importance"]
        Sf = Sc + Ni
        cfg = _cfg_struct(cfgd, ray_batch.shape[1])
        records = isinstance(path, _TcTrain)
        pc, pf = net_c.net_params(), (net_f.net_params() if net_f is not None else None)
        pk_c = _packed_for(net_c, cfg.precision)
        pk_f = _packed_for(net_f, cfg.precision) if net_f is not None else None
        if records:                                 # the training forward reads its path's image
            pk_c, pk_f = path.image(net_c), (path.image(net_f) if net_f is not None else None)
        f32 = dict(device=dev, dtype=torch.float32)
        t_vals = _linspace01(Sc, dev)                                             # run_nerf.py:357
        u_det = _linspace01(Ni, dev) if Ni > 0 else None                          # run_nerf_helpers.py:205
        z_c = torch.empty((N, Sc), **f32)
        o = {k: torch.empty(s, **f32) for k, s in (("rgb0", (N, 3)), ("disp0", (N,)), ("acc0", (N,)), ("w0", (N, Sc)))}
        retraw, fine = cfgd["retraw"], Ni > 0
        # raw is kept outside tc_fp16 (tc_split runs like fp32 here unless it trains on records) and for the records' backward
        keep_raw = cfg.precision != PREC_TC_FP16 or records
        raw_c = torch.empty((N, Sc, 4), **f32) if ((retraw and not fine) or keep_raw) else None
        out_c = NerfPassOut(_ptr(o["rgb0"]), _ptr(o["disp0"]), _ptr(o["acc0"]), C.c_void_p(0), _ptr(o["w0"]), _ptr(raw_c))
        z_f = z_std = raw_f = None
        out_f = None
        if fine:
            z_f, z_std = torch.empty((N, Sf), **f32), torch.empty((N,), **f32)
            o.update(rgb=torch.empty((N, 3), **f32), disp=torch.empty((N,), **f32), acc=torch.empty((N,), **f32))
            raw_f = torch.empty((N, Sf, 4), **f32) if (retraw or keep_raw) else None
            out_f = NerfPassOut(_ptr(o["rgb"]), _ptr(o["disp"]), _ptr(o["acc"]), C.c_void_p(0), C.c_void_p(0), _ptr(raw_f))
        ws_bytes = lib.nerf_b200_march_workspace_bytes(N, Sf)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        common = (_ptr(ray_batch), N, C.byref(cfg), C.byref(pc), _ptr(pk_c), C.byref(pf) if pf is not None else None, _ptr(pk_f),
                  _ptr(t_vals), _ptr(u_det), _ptr(t_rand), _ptr(u_rand), _ptr(noise0), _ptr(noise1),
                  _ptr(z_c), C.byref(out_c), _ptr(z_f), _ptr(z_std), C.byref(out_f) if out_f is not None else None,
                  _ptr(ws), ws_bytes)
        saved_rec = ()
        # render() may have left the construction of this very batch to the prologue launch (_DEFERRED_PACK): take it over here
        gen = _take_deferred_pack(ray_batch)
        with _on(ray_batch):
            if records:
                if gen is not None:                 # the training-mode entry builds nothing: one extra launch now
                    _launch_pack(lib, gen, ray_batch)
                sv_c, act_c, mask_c = _train_save(lib, N, Sc, pc, dev, path)
                saved_rec = (raw_c, act_c, mask_c)
                sv_f = None
                if fine:
                    sv_f, act_f, mask_f = _train_save(lib, N, Sf, pf if pf is not None else pc, dev, path)
                    saved_rec += (raw_f, act_f, mask_f)
                _call(lib, path.fwd, *common, C.byref(sv_c), C.byref(sv_f) if sv_f is not None else None, _stream(ray_batch))
            elif gen is not None:
                check(lib.nerf_b200_render_fwd(C.byref(gen[0]), *common, _stream(ray_batch)), "render_fwd")
            else:
                check(lib.nerf_b200_render_rays_fwd(*common, _stream(ray_batch)), "render_rays_fwd")
        if ctx is not None:
            ctx.cfgd, ctx.path, ctx.nets = cfgd, path, (net_c, net_f)
            ctx.save_for_backward(ray_batch, z_c, z_f if fine else torch.empty(0, device=dev),
                                  noise0 if noise0 is not None else torch.empty(0, device=dev),
                                  noise1 if noise1 is not None else torch.empty(0, device=dev), *saved_rec)
        # as in the reference every map and raw carry a gradient; z_std does not (z_samples is detached, :394)
        if fine:
            rets = (o["rgb"], o["disp"], o["acc"], o["rgb0"], o["disp0"], o["acc0"], z_std,
                    raw_f if retraw else torch.empty(0, device=dev))
            if ctx is not None:
                ctx.mark_non_differentiable(z_std, *(() if retraw else (rets[7],)))
        else:
            rets = (o["rgb0"], o["disp0"], o["acc0"], raw_c if retraw else torch.empty(0, device=dev))
            if ctx is not None and not retraw:
                ctx.mark_non_differentiable(rets[3])
        if ctx is not None:
            ctx.set_materialize_grads(False)
        return rets

    @staticmethod
    def backward(ctx, *g):
        lib = _lib.load()
        ray_batch, z_c, z_f, noise0, noise1 = ctx.saved_tensors[:5]
        rec = ctx.saved_tensors[5:]
        fine = ctx.cfgd["N_importance"] > 0
        N = ray_batch.shape[0]
        cfg = _cfg_struct(ctx.cfgd, ray_batch.shape[1])
        # seeds per pass: fine <- rgb, disp, acc, raw;  coarse <- rgb0, disp0, acc0 (and raw without fine samples)
        if fine:
            s_fine = dict(rgb_map=g[0], disp_map=g[1], acc_map=g[2], raw=g[7])
            s_coarse = dict(rgb_map=g[3], disp_map=g[4], acc_map=g[5])
        else:
            s_fine, s_coarse = {}, dict(rgb_map=g[0], disp_map=g[1], acc_map=g[2], raw=g[3])
        # the split path has no rgb-only entries: its seeds are NerfOutGrads, and a pass without one is skipped
        rgb_only = (ctx.path == "exact" or ctx.path.bwd_rgb is not None) and \
            not any(v is not None for s in (s_fine, s_coarse) for k, v in s.items() if k != "rgb_map")

        def seed(s):
            if not rgb_only:
                return _out_grads(**s) if any(v is not None for v in s.values()) else None
            g_rgb = s["rgb_map"]
            if g_rgb is None and fine:                  # both passes run: an unused rgb output seeds zeros
                g_rgb = torch.zeros((N, 3), device=ray_batch.device)
            return None if g_rgb is None else g_rgb.contiguous().float()
        return _RenderRays._backward(ctx, lib, ray_batch, z_c, z_f, noise0, noise1, rec, cfg,
                                     seed(s_fine) if fine else None, seed(s_coarse), rgb_only)

    @staticmethod
    def _passes(ctx, z_c, z_f, noise0, noise1, rec, seed_f, seed_c):
        """[(seed, z, noise or None, net, grad buffers, records)] of the coarse and (with fine samples) the fine pass, and the
        parameter gradients autograd receives."""
        net_c, net_f = ctx.nets
        fine = ctx.cfgd["N_importance"] > 0
        grads_c = _grad_buffers(net_c)
        same_net = fine and (net_f is None)
        grads_f = grads_c if same_net else (_grad_buffers(net_f) if fine else None)
        passes = [(seed_c, z_c, noise0 if noise0.numel() else None, net_c, grads_c, rec[0:3])]
        if fine:
            passes.append((seed_f, z_f, noise1 if noise1.numel() else None, net_c if same_net else net_f, grads_f, rec[3:6]))
        out = [None] * 9
        out += [grads_c[k] for _, _, k, _ in net_c._named_params()]
        if net_f is not None:
            out += [grads_f[k] for _, _, k, _ in net_f._named_params()]
        return passes, tuple(out)

    @staticmethod
    def _backward(ctx, lib, ray_batch, z_c, z_f, noise0, noise1, rec, cfg, seed_f, seed_c, rgb_only):
        """The backward of the passes with a seed (None: the pass does not run).  rgb_only: each seed is dL/drgb_map and the
        rgb-only entry points run; otherwise each seed is a (NerfOutGrads, tensors) pair from _out_grads and the NerfOutGrads
        entry points run.  A tensor-core path runs both passes in one call (one after the other on the stream) when both
        have a seed, else the pass that has one; the exact path runs each pass that has one."""
        N, path = ray_batch.shape[0], ctx.path

        def seed_arg(seed):
            return _ptr(seed) if rgb_only else C.byref(seed[0])
        passes, out = _RenderRays._passes(ctx, z_c, z_f, noise0, noise1, rec, seed_f, seed_c)
        passes = [p for p in passes if p[0] is not None]
        with _on(ray_batch):
            if path == "exact":
                for seed, z, noise, net, gbuf, _ in passes:
                    n, gs, S = net.net_params(), net.grad_struct(gbuf), z.shape[1]
                    ws_bytes = lib.nerf_b200_march_bwd_workspace_bytes(N, S, C.byref(n))
                    ws = _workspace(ws_bytes, z.device)
                    _call(lib, "nerf_b200_march_bwd" if rgb_only else "nerf_b200_march_bwd_outs", _ptr(ray_batch), _ptr(z), _ptr(noise),
                          N, S, C.byref(n), _ptr(None), C.byref(cfg), seed_arg(seed), C.byref(gs), _ptr(ws), ws_bytes, _stream(z))
                return out
            bp = [_bwd_pass(z, noise, z.shape[1], net.net_params(), path.image(net), rc[0], _records_save(rc[1], rc[2]),
                            seed if rgb_only else None, net.grad_struct(gbuf)) for seed, z, noise, net, gbuf, rc in passes]
            if len(bp) == 2:
                ws_bytes = getattr(lib, path.bwd_ws)(N, bp[0].S, bp[0].net, bp[1].S, bp[1].net)
                ws = _workspace(ws_bytes, ray_batch.device)
                seeds = () if rgb_only else (C.byref(seed_c[0]), C.byref(seed_f[0]))
                _call(lib, path.bwd_rgb if rgb_only else path.bwd, _ptr(ray_batch), N, C.byref(cfg), C.byref(bp[0]), C.byref(bp[1]),
                      *seeds, _ptr(ws), ws_bytes, _stream(ray_batch))
            elif bp:
                (q,), seed = bp, passes[0][0]
                ws_bytes = getattr(lib, path.march_bwd_ws)(N, q.S, q.net)
                ws = _workspace(ws_bytes, ray_batch.device)
                _call(lib, path.march_bwd_rgb if rgb_only else path.march_bwd, _ptr(ray_batch), q.z_vals, q.noise, N, q.S, q.net, q.packed,
                      C.byref(cfg), q.raw, q.save, seed_arg(seed), q.grads, _ptr(ws), ws_bytes, _stream(ray_batch))
        return out


def render_rays(ray_batch, network_fn, network_query_fn, N_samples, retraw=False, lindisp=False, perturb=0.,
                N_importance=0, network_fine=None, white_bkgd=False, raw_noise_std=0., verbose=False, pytest=False):
    """Volumetric rendering of one ray chunk; same contract as run_nerf.py:308-418.

    Returns rgb_map, disp_map, acc_map, [raw], and with N_importance > 0 rgb0, disp0, acc0, z_std.
    The reference's NaN/Inf scan (:414-416, 16 host syncs per call) is only run when DEBUG is set."""
    ray_batch = _f32c(ray_batch, "ray_batch")
    if not isinstance(network_fn, NeRF) or (network_fine is not None and not isinstance(network_fine, NeRF)):
        raise RuntimeError("nerf_b200.render_rays: networks must be nerf_b200.NeRF modules")
    N = ray_batch.shape[0]
    dev = ray_batch.device
    use_viewdirs = ray_batch.shape[-1] > 8
    if use_viewdirs != bool(network_fn.use_viewdirs):
        raise RuntimeError("ray batch / network disagree on use_viewdirs")
    mr = getattr(network_query_fn, "multires", None)
    if mr is None:
        # a foreign closure: recover L from the module's input widths
        mr, mrv = (network_fn.input_ch - 3) // 6, (network_fn.input_ch_views - 3) // 6 if use_viewdirs else 0
    else:
        mrv = network_query_fn.multires_views
    if N == 0:
        e = lambda *s: torch.empty(s, device=dev)
        ret = {"rgb_map": e(0, 3), "disp_map": e(0), "acc_map": e(0)}
        if retraw:
            ret["raw"] = e(0, N_samples + N_importance, 4)
        if N_importance > 0:
            ret.update(rgb0=e(0, 3), disp0=e(0), acc0=e(0), z_std=e(0))
        return ret
    t_rand = u_rand = None
    if perturb > 0.:                                                              # run_nerf.py:365-377
        if pytest:
            np.random.seed(0)
            t_rand = torch.tensor(np.random.rand(N, N_samples), dtype=torch.float32, device=dev)
        else:
            t_rand = torch.rand(N, N_samples, device=dev)
    # draw order of the reference (a seeded run consumes the generator alike): t_rand :371, coarse noise :285, u :208, fine noise :285
    noise0 = _draw_noise((N, N_samples), float(raw_noise_std), pytest, dev)
    if perturb > 0. and N_importance > 0:
        u_rand, _ = _draw_u((N, N_importance), False, pytest, dev)               # det = (perturb == 0), :393
    noise1 = _draw_noise((N, N_samples + N_importance), float(raw_noise_std), pytest, dev) if N_importance > 0 else None
    cfgd = dict(N_samples=int(N_samples), N_importance=int(N_importance), multires=int(mr), multires_views=int(mrv),
                lindisp=bool(lindisp), perturb=float(perturb), white_bkgd=bool(white_bkgd), retraw=bool(retraw))
    net_f = network_fine if N_importance > 0 else None          # the reference ignores network_fine without fine samples
    params = [q for _, _, _, q in network_fn._named_params()] + ([q for _, _, _, q in net_f._named_params()] if net_f is not None else [])
    # gradients are needed when grad mode is on AND a parameter requires one (inside Function.forward grad mode is always off,
    # and ctx.needs_input_grad stays True under torch.no_grad())
    path = _train_path(get_precision(), get_backward(), torch.is_grad_enabled() and any(p.requires_grad for p in params), network_fn, net_f)
    if path is not None:
        outs = _RenderRays.apply(ray_batch, cfgd, path, network_fn, net_f, t_rand, u_rand, noise0, noise1, *params)
    else:                                                        # inference: no autograd node to build (saves ~50 us of host time per call)
        with torch.no_grad():
            outs = _RenderRays.forward(None, ray_batch, cfgd, None, network_fn, net_f, t_rand, u_rand, noise0, noise1)
    if N_importance > 0:
        rgb, disp, acc, rgb0, disp0, acc0, z_std, raw = outs
        ret = {"rgb_map": rgb, "disp_map": disp, "acc_map": acc}
        if retraw:
            ret["raw"] = raw
        ret.update(rgb0=rgb0, disp0=disp0, acc0=acc0, z_std=z_std)
    else:
        rgb, disp, acc, raw = outs
        ret = {"rgb_map": rgb, "disp_map": disp, "acc_map": acc}
        if retraw:
            ret["raw"] = raw
    if DEBUG:
        for k in ret:
            if torch.isnan(ret[k]).any() or torch.isinf(ret[k]).any():
                print(f"! [Numerical Error] {k} contains nan or inf.")
    return ret


def batchify_rays(rays_flat, chunk=1024 * 32, **kwargs):
    """run_nerf.py:54-66."""
    all_ret = {}
    for i in range(0, rays_flat.shape[0], chunk):
        ret = render_rays(rays_flat[i:i + chunk], **kwargs)
        for k in ret:
            all_ret.setdefault(k, []).append(ret[k])
    return {k: (torch.cat(v, 0) if len(v) > 1 else v[0]) for k, v in all_ret.items()}


def _camera(H, W, K, c2w=None) -> NerfCamera:
    cam = NerfCamera()
    cam.H, cam.W = int(H), int(W)
    cam.fx, cam.fy, cam.cx, cam.cy = float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2])
    if c2w is not None:
        m = c2w.detach().float().cpu().numpy() if torch.is_tensor(c2w) else np.asarray(c2w, np.float32)
        for i, v in enumerate(np.ascontiguousarray(m[:3, :4], np.float32).reshape(-1)):
            cam.c2w[i] = float(v)
    return cam


def _render_device(kwargs):
    net = kwargs.get("network_fn")
    return net._check_device() if isinstance(net, NeRF) else torch.device("cuda")


def _is_scalar(x):
    """Python / numpy scalar (np.float32 near/far of the LLFF and deepvoxels loaders included), not a tensor."""
    return not torch.is_tensor(x) and np.ndim(x) == 0 and isinstance(x, (numbers.Real, np.generic))


def render(H, W, K, chunk=1024 * 32, rays=None, c2w=None, ndc=True, near=0., far=1., use_viewdirs=False,
           c2w_staticcam=None, **kwargs):
    """run_nerf.py:69-134: build the [N, 8|11] ray batch, render in `chunk`-ray slices, reshape.

    The batch construction -- get_rays for `c2w` (run_nerf_helpers.py:153-162), view-direction normalisation (:108),
    NDC warp (run_nerf_helpers.py:175-192), near/far and packing (:117-123) -- is one kernel (nerf_b200_pack_rays) in
    every mode, `c2w_staticcam` (rays from one camera, view directions from another, :104-107) included; per-ray
    near/far arrays are written into their two columns afterwards."""
    lib = _lib.load()
    net_c, net_f = kwargs.get("network_fn"), kwargs.get("network_fine")
    want = torch.is_grad_enabled() and any(p.requires_grad for n in (net_c, net_f) if isinstance(n, nn.Module) for p in n.parameters())
    net_f = net_f if kwargs.get("N_importance", 0) > 0 else None
    # refuse what cannot train before the batch is built; networks that are not NeRF modules are render_rays' to refuse
    nets = (net_c, net_f) if isinstance(net_c, NeRF) and (net_f is None or isinstance(net_f, NeRF)) else ()
    _train_path(get_precision(), get_backward(), want, *nets)
    if get_precision() == "fp32":                  # refuse a net the exact path cannot run before the batch is built
        for net in (net_c, net_f):
            if isinstance(net, NeRF) and lib.nerf_b200_march_bwd_workspace_bytes(1, 1, C.byref(net.net_params())) == 0:
                raise RuntimeError("nerf_b200: " + lib.nerf_b200_last_error().decode())
    ndc = int(bool(ndc))
    if c2w is not None:
        dev = _render_device(kwargs)
        N, sh = int(H) * int(W), [int(H), int(W), 3]
        given = None
    else:
        rays_o, rays_d = rays
        sh = list(rays_d.shape)
        given = (_f32c(rays_o, "rays_o").reshape(-1, 3), _f32c(rays_d, "rays_d").reshape(-1, 3))
        dev, N = given[0].device, given[0].shape[0]
    scalar_bounds = _is_scalar(near) and _is_scalar(far)
    nf = (float(near), float(far)) if scalar_bounds else (0., 1.)
    packed = torch.empty((N, 11 if use_viewdirs else 8), device=dev, dtype=torch.float32)

    # one chunk, scalar bounds, one camera: the batch is built by render_rays' own prologue launch (see _DEFERRED_PACK)
    defer = scalar_bounds and c2w_staticcam is None and N <= chunk and get_precision() in ("tc_fp16", "tc_split")

    def pack(o, d, view_src, cam, out, ndc_, viewdirs_):
        global _DEFERRED_PACK
        if defer and out is packed:
            _flush_deferred_pack()
            gen = _lib.NerfRayGen(_ptr(o), _ptr(d), _ptr(view_src), C.pointer(cam), 0, ndc_, int(bool(viewdirs_)), nf[0], nf[1])
            _DEFERRED_PACK = (packed, (gen, cam, o, d, view_src))
            return
        check(lib.nerf_b200_pack_rays(_ptr(o), _ptr(d), _ptr(view_src), C.byref(cam), N, 0, ndc_, nf[0], nf[1], int(bool(viewdirs_)),
                                      _ptr(out), _stream(out)), "pack_rays")

    with _on(packed):
        view_src = None
        if c2w_staticcam is not None:
            # view directions come from the `c2w` / given rays, the rays themselves from the static camera (:104-107)
            if use_viewdirs:
                if given is not None:
                    view_src = given[1]
                else:
                    tmp = torch.empty((N, 8), device=dev, dtype=torch.float32)
                    pack(None, None, None, _camera(H, W, K, c2w), tmp, 0, False)
                    view_src = tmp[:, 3:6].contiguous()
            pack(None, None, view_src, _camera(H, W, K, c2w_staticcam), packed, ndc, use_viewdirs)
        elif given is None:
            pack(None, None, None, _camera(H, W, K, c2w), packed, ndc, use_viewdirs)
        else:
            pack(given[0], given[1], None, _camera(H, W, K), packed, ndc, use_viewdirs)
    if not scalar_bounds:                                                          # :117-118 with array bounds
        shape_col = lambda x: torch.as_tensor(x, dtype=torch.float32, device=dev).expand(N) if np.ndim(x) == 0 or (torch.is_tensor(x) and x.dim() == 0) \
            else torch.as_tensor(x, dtype=torch.float32, device=dev).reshape(N)
        packed[:, 6] = shape_col(near)
        packed[:, 7] = shape_col(far)
    try:
        all_ret = batchify_rays(packed, chunk, **kwargs)
    finally:
        _flush_deferred_pack()                                # (only if the forward never saw the batch: an exception on the way)
    for k in all_ret:
        all_ret[k] = torch.reshape(all_ret[k], list(sh[:-1]) + list(all_ret[k].shape[1:]))
    k_extract = ["rgb_map", "disp_map", "acc_map"]
    return [all_ret[k] for k in k_extract] + [{k: all_ret[k] for k in all_ret if k not in k_extract}]


def render_to8b(H, W, K, c2w, chunk=1024 * 32, out=None, **kwargs):
    """One frame of render_path (run_nerf.py:151-169) with the image output on the device: rays are generated per chunk from
    the camera (pixel offset, no [H,W,3] ray tensors), rendered, converted with to8b (run_nerf_helpers.py:11) by a kernel and
    copied to pinned host memory asynchronously.  Returns (rgb8 [H,W,3] uint8 pinned host tensor, disp [H,W] float32 CUDA
    tensor); synchronise the stream (or call .numpy() after torch.cuda.synchronize()) before reading rgb8.  No reference
    counterpart in signature; `kwargs` are render()'s (render_kwargs_test + near/far + ndc/use_viewdirs)."""
    lib = _lib.load()
    dev = _render_device(kwargs)
    kw = dict(kwargs)
    ndc, use_viewdirs = int(bool(kw.pop("ndc", True))), bool(kw.pop("use_viewdirs", False))
    near, far = float(kw.pop("near", 0.)), float(kw.pop("far", 1.))
    n_pix = int(H) * int(W)
    cam = _camera(H, W, K, c2w)
    rgb8_dev = torch.empty((n_pix, 3), dtype=torch.uint8, device=dev)
    disp = torch.empty((n_pix,), dtype=torch.float32, device=dev)
    host = out if out is not None else torch.empty((int(H), int(W), 3), dtype=torch.uint8, device="cpu").pin_memory()
    with torch.no_grad(), _on(rgb8_dev):
        for p0 in range(0, n_pix, chunk):
            n = min(chunk, n_pix - p0)
            packed = torch.empty((n, 11 if use_viewdirs else 8), device=dev, dtype=torch.float32)
            check(lib.nerf_b200_pack_rays(None, None, None, C.byref(cam), n, p0, ndc, near, far, int(use_viewdirs), _ptr(packed), _stream(packed)), "pack_rays")
            ret = render_rays(packed, **kw)
            rgb = ret["rgb_map"].contiguous()
            check(lib.nerf_b200_to8b(_ptr(rgb), n * 3, _ptr(rgb8_dev[p0:p0 + n]), _stream(rgb)), "to8b")
            disp[p0:p0 + n] = ret["disp_map"]
        host.view(-1, 3).copy_(rgb8_dev, non_blocking=True)
    return host, disp.view(int(H), int(W))


class DeviceRayBatcher:
    """The two ray-batching modes of train() (run_nerf.py:677-757) with the data resident on the device (SURVEY 8f rank 3).

    use_batching=True : `rays_rgb` [(N_img*H*W), 3, 3] (ro, rd, rgb) lives on the device, is shuffled with torch.randperm at every
                        epoch end (:746-750) and sliced; next() -> (batch_rays [2,B,3], target [B,3]).  As in the reference's
                        slicing (:717-726), the last batch of an epoch is shorter when the ray count is not a multiple of B:
                        it holds the remaining n < B rays.  FusedTrainStep takes it on the first n rows of its buffers
                        (step.rays[:, :n], step.target[:n], step_device(n_rays=n); INTEGRATION §5a).
    use_batching=False: per step one random training image; pixel ids are drawn on the device (inside the centre crop while
                        i < precrop_iters, :731-744) and the targets gathered there; next() -> (c2w [3,4], pixel_index [B] int64,
                        target [B,3]) for FusedTrainStep.step_device(c2w, pixel_index) / nerf_b200_pack_rays_pixels."""

    def __init__(self, images, poses, H, W, N_rand, i_train=None, rays_rgb=None, precrop_iters=0, precrop_frac=0.5, device="cuda"):
        self.dev = torch.device(device)
        self.H, self.W, self.B = int(H), int(W), int(N_rand)
        self.images = torch.as_tensor(images, dtype=torch.float32, device=self.dev)
        self.poses = torch.as_tensor(poses, dtype=torch.float32)                        # host: one [3,4] pose per step goes into kernel arguments
        self.i_train = list(range(self.images.shape[0])) if i_train is None else [int(i) for i in i_train]
        self.rays_rgb = None if rays_rgb is None else torch.as_tensor(rays_rgb, dtype=torch.float32, device=self.dev)
        # self.rays_rgb == the constructor's rays_rgb[self.perm]: the order to restore, without saving the shuffled rays
        self.perm = None if rays_rgb is None else torch.arange(self.rays_rgb.shape[0], device=self.dev)
        self.i_batch, self.step = 0, 0
        self.precrop_iters, self.precrop_frac = int(precrop_iters), float(precrop_frac)

    def next(self):
        self.step += 1
        if self.rays_rgb is not None:
            b = self.rays_rgb[self.i_batch:self.i_batch + self.B].transpose(0, 1)
            self.i_batch += self.B
            if self.i_batch >= self.rays_rgb.shape[0]:
                idx = torch.randperm(self.rays_rgb.shape[0], device=self.dev)
                self.rays_rgb, self.perm = self.rays_rgb[idx], self.perm[idx]
                self.i_batch = 0
            return b[:2].contiguous(), b[2].contiguous()
        img_i = self.i_train[int(torch.randint(len(self.i_train), (1,)).item())]
        if self.step <= self.precrop_iters:
            dH, dW = int(self.H // 2 * self.precrop_frac), int(self.W // 2 * self.precrop_frac)
            j = torch.randint(self.H // 2 - dH, self.H // 2 + dH, (self.B,), device=self.dev)
            i = torch.randint(self.W // 2 - dW, self.W // 2 + dW, (self.B,), device=self.dev)
            pix = j * self.W + i
        else:
            pix = torch.randperm(self.H * self.W, device=self.dev)[:self.B]             # np.random.choice(..., replace=False), :741
        target = self.images[img_i].reshape(-1, self.images.shape[-1])[pix][:, :3].contiguous()
        return self.poses[img_i][:3, :4], pix, target

    def state_dict(self):
        """The batcher's position: `step` (which decides the centre crop), `i_batch`, the state of the host's torch generator (the
        image draw of no_batching) and, with use_batching, the current order of rays_rgb as an int64 permutation of the
        constructor's rays_rgb (8 bytes per ray instead of the 36 of the shuffled rays).  The device draws (the epoch-end
        randperm, the pixel ids) come from the CUDA generator, which FusedTrainStep.state_dict() holds."""
        return {"step": self.step, "i_batch": self.i_batch, "cpu_rng_state": torch.get_rng_state(),
                "perm": None if self.perm is None else self.perm.cpu()}

    def load_state_dict(self, sd):
        """The inverse of state_dict(), on a batcher constructed with the same images, poses, rays_rgb and settings.  It also
        sets the host's torch generator (torch.set_rng_state), from which next() draws the image of no_batching."""
        perm = sd["perm"]
        if (perm is None) != (self.rays_rgb is None):
            raise RuntimeError("DeviceRayBatcher.load_state_dict: the state is of the other batching mode (use_batching differs)")
        if perm is not None:
            n = self.rays_rgb.shape[0]
            perm = perm.to(self.dev)
            if perm.dtype != torch.int64 or tuple(perm.shape) != (n,) or \
                    not torch.equal(torch.sort(perm).values, torch.arange(n, device=self.dev)):
                raise RuntimeError(f"DeviceRayBatcher.load_state_dict: 'perm' is not an int64 permutation of this batcher's {n} rays")
            if not 0 <= int(sd["i_batch"]) < n:
                raise RuntimeError(f"DeviceRayBatcher.load_state_dict: i_batch {int(sd['i_batch'])} is outside [0, {n})")
            inv = torch.empty_like(self.perm)
            inv[self.perm] = torch.arange(n, device=self.dev)
            self.rays_rgb, self.perm = self.rays_rgb[inv[perm]], perm
        self.step, self.i_batch = int(sd["step"]), int(sd["i_batch"])
        torch.set_rng_state(sd["cpu_rng_state"].cpu())


# ------------------------------------------------------------------------------------------------
# create_nerf  (run_nerf.py:178-259)
# ------------------------------------------------------------------------------------------------

def create_nerf(args, device=None):
    """Instantiate NeRF's MLP models, optimizer and render kwargs; same 5-tuple as the reference."""
    device = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
    embed_fn, input_ch = get_embedder(args.multires, args.i_embed)
    input_ch_views, embeddirs_fn = 0, None
    if args.use_viewdirs:
        embeddirs_fn, input_ch_views = get_embedder(args.multires_views, args.i_embed)
    output_ch = 5 if args.N_importance > 0 else 4
    skips = [4]
    model = NeRF(D=args.netdepth, W=args.netwidth, input_ch=input_ch, output_ch=output_ch, skips=skips,
                 input_ch_views=input_ch_views, use_viewdirs=args.use_viewdirs).to(device)
    grad_vars = list(model.parameters())
    model_fine = None
    if args.N_importance > 0:
        model_fine = NeRF(D=args.netdepth_fine, W=args.netwidth_fine, input_ch=input_ch, output_ch=output_ch,
                          skips=skips, input_ch_views=input_ch_views, use_viewdirs=args.use_viewdirs).to(device)
        grad_vars += list(model_fine.parameters())
    network_query_fn = _QueryFn(embed_fn, embeddirs_fn, args.netchunk, args.multires, args.multires_views, args.i_embed)
    optimizer = torch.optim.Adam(params=grad_vars, lr=args.lrate, betas=(0.9, 0.999))
    start = 0
    basedir, expname = args.basedir, args.expname
    if args.ft_path is not None and args.ft_path != 'None':
        ckpts = [args.ft_path]
    else:
        ckpts = [os.path.join(basedir, expname, f) for f in sorted(os.listdir(os.path.join(basedir, expname))) if 'tar' in f]
    print('Found ckpts', ckpts)
    if len(ckpts) > 0 and not args.no_reload:
        ckpt_path = ckpts[-1]
        print('Reloading from', ckpt_path)
        ckpt = torch.load(ckpt_path, map_location=device)
        start = ckpt['global_step']
        optimizer.load_state_dict(ckpt['optimizer_state_dict'])
        model.load_state_dict(ckpt['network_fn_state_dict'])
        if model_fine is not None:
            model_fine.load_state_dict(ckpt['network_fine_state_dict'])
    render_kwargs_train = {
        'network_query_fn': network_query_fn, 'perturb': args.perturb, 'N_importance': args.N_importance,
        'network_fine': model_fine, 'N_samples': args.N_samples, 'network_fn': model,
        'use_viewdirs': args.use_viewdirs, 'white_bkgd': args.white_bkgd, 'raw_noise_std': args.raw_noise_std,
    }
    if args.dataset_type != 'llff' or args.no_ndc:
        print('Not ndc!')
        render_kwargs_train['ndc'] = False
        render_kwargs_train['lindisp'] = args.lindisp
    render_kwargs_test = {k: render_kwargs_train[k] for k in render_kwargs_train}
    render_kwargs_test['perturb'] = False
    render_kwargs_test['raw_noise_std'] = 0.
    return render_kwargs_train, render_kwargs_test, start, grad_vars, optimizer



# ------------------------------------------------------------------------------------------------
# CUDA-graph replay of render() for up to a fixed ray count (no reference counterpart)
# ------------------------------------------------------------------------------------------------

def _capture_graph(dev, warm_up, body, pool=None, keep_rng=False):
    """Run `warm_up()` on a side stream, so that one-time work (weight packing, opt-ins, caches, lazy initialisations) stays
    out of the capture, then capture `body()` into a new CUDA graph -> (graph, what body returned).  `pool`: the memory pool
    of an earlier graph (`graph.pool()`) to allocate from, for graphs that never run concurrently.  `keep_rng`: put the
    device's CUDA generator back to its state before the warm-up, so that a capture made in the middle of a run leaves every
    later random draw as it would have been without it (the capture itself draws nothing)."""
    rng = torch.cuda.get_rng_state(dev) if keep_rng else None
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        warm_up()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    if rng is not None:
        torch.cuda.set_rng_state(rng, dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, pool=pool):
        out = body()
    return graph, out


class GraphedRender:
    """`render(H, W, K, rays=..., **render_kwargs)` under `torch.no_grad()`, captured into a CUDA graph and replayed per
    call: host -> device copy of the rays, one graph launch (ray packing, z sampling, both fused passes, resampling), one
    device -> host copy of `[rgb(3), disp, acc]`.

    `n_rays` is the capacity: a call takes any n <= n_rays rays, such as the tail chunk of a frame that is not a whole number
    of chunks.  The constructor captures n_rays; every other n is captured on its first call, as
    `render(H, W, K, rays=self.rays[:, :n], ...)` in the first graph's memory pool, and kept.

    After the fusion a 4096-ray render is ~1 ms of GPU time, so the ~10 Python-level launches and allocations of
    `render()` (the reference's structure, run_nerf.py:69-134 -> :54-66 -> :308-418) cost as much as the kernels
    when the GPU starts idle; render_only / test-time callers (run_nerf.py:668,:805,:823 iterate `render` over
    poses under no_grad) can use this instead.  Deterministic settings only (perturb = 0, raw_noise_std = 0:
    the graph would replay the same random draws).  Weight updates are picked up by `refresh()` (re-packs into
    the same device buffer the graphs read)."""

    def __init__(self, H, W, K, n_rays, **render_kwargs):
        if render_kwargs.get("perturb", 0.) or render_kwargs.get("raw_noise_std", 0.):
            raise ValueError("GraphedRender supports deterministic rendering only (perturb = 0, raw_noise_std = 0)")
        self._nets = [n for n in (render_kwargs.get("network_fn"), render_kwargs.get("network_fine")) if isinstance(n, NeRF)]
        self.n_rays = int(n_rays)
        self.rays = torch.zeros((2, self.n_rays, 3), device=_render_device(render_kwargs), dtype=torch.float32)
        self.rays[1, :, 2] = -1.0                                       # any non-degenerate direction for the warm-up
        self.host_out = torch.empty((self.n_rays, 5), dtype=torch.float32, device="cpu").pin_memory()
        self._render = lambda rays: render(H, W, K, rays=rays, **render_kwargs)
        self.graph = None
        self._graphs = {}                       # n -> (graph, packed_out, device_out, self.rays[:, :n], self.host_out[:n])
        self.graph, self.packed_out, self.device_out = self._graph(self.n_rays)[:3]

    def _graph(self, n):
        if n not in self._graphs:
            rays = self.rays[:, :n]

            def body():
                rgb, disp, acc, extras = self._render(rays)
                return torch.cat([rgb, disp[:, None], acc[:, None]], -1), (rgb, disp, acc, extras)
            with torch.no_grad():
                graph, (packed, dev_out) = _capture_graph(self.rays.device, lambda: [self._render(rays) for _ in range(2)], body,
                                                          pool=None if self.graph is None else self.graph.pool())
            self._graphs[n] = (graph, packed, dev_out, rays, self.host_out[:n])
        return self._graphs[n]

    def refresh(self):
        """Call after the networks' parameters changed (optimizer step, load_state_dict)."""
        for n in self._nets:
            _packed_for(n, _PRECISION["mode"])

    def __call__(self, rays_host):
        """rays_host: [2, n, 3] fp32 with 0 < n <= n_rays (pinned memory makes the copy asynchronous).  Returns the first n
        rows of the pinned host tensor `host_out` [n_rays, 5] = rgb_map (3), disp_map, acc_map; the device tensors of the
        last call stay available in `.device_out`.  Synchronises the current stream before returning."""
        sh = tuple(rays_host.shape)
        if len(sh) != 3 or sh[0] != 2 or sh[2] != 3 or not 0 < sh[1] <= self.n_rays:
            raise RuntimeError(f"GraphedRender: rays of shape {sh}; expected [2, n, 3] with 0 < n <= {self.n_rays}")
        graph, self.packed_out, self.device_out, rays, out = self._graph(sh[1])
        rays.copy_(rays_host, non_blocking=True)
        graph.replay()
        out.copy_(self.packed_out, non_blocking=True)
        torch.cuda.current_stream(self.rays.device).synchronize()
        return out


# ------------------------------------------------------------------------------------------------
# mesh extraction: the density over a grid and marching cubes on it
# ------------------------------------------------------------------------------------------------

def _axis(a, what, dev=None):
    a = _f32c(torch.as_tensor(a, device=dev) if not torch.is_tensor(a) else a, what).reshape(-1)
    if dev is not None and a.device != dev:
        raise RuntimeError(f"nerf_b200: {what} is on {a.device}, expected {dev}")
    return a


@torch.no_grad()
def density_grid(network_fn, network_query_fn, xs, ys, zs):
    """sigma [nx, ny, nz] (float32, on xs' device) of `network_fn` at the points (xs[i], ys[j], zs[k]), in the current
    set_precision: bit for bit run_network(torch.meshgrid(xs, ys, zs, indexing='ij'), zero viewdirs)[..., 3], the pre-ReLU
    density without noise, but without materialising the points or evaluating the view layers.  `multires` is read from
    `network_query_fn` as render_rays reads it."""
    if not isinstance(network_fn, NeRF):
        raise RuntimeError("nerf_b200.density_grid: network must be a nerf_b200.NeRF")
    xs = _axis(xs, "xs")
    ys, zs = _axis(ys, "ys", xs.device), _axis(zs, "zs", xs.device)
    mr = getattr(network_query_fn, "multires", None)
    if mr is None:
        mr = (network_fn.input_ch - 3) // 6
    nx, ny, nz = xs.numel(), ys.numel(), zs.numel()
    lib = _lib.load()
    n = network_fn.net_params()
    prec = _PRECISION["mode"]
    packed = _packed_for(network_fn, prec)
    sigma = torch.empty((nx, ny, nz), device=xs.device, dtype=torch.float32)
    ws_bytes = lib.nerf_b200_density_grid_workspace_bytes(nx, ny, nz, C.byref(n), prec)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=xs.device)
    with _on(xs):
        check(lib.nerf_b200_density_grid(_ptr(xs), nx, _ptr(ys), ny, _ptr(zs), nz, C.byref(n), _ptr(packed), int(mr), prec,
                                         _ptr(sigma), _ptr(ws), ws_bytes, _stream(xs)), "density_grid")
    return sigma


@torch.no_grad()
def marching_cubes(sigma, xs, ys, zs, iso):
    """Marching cubes of sigma [nx, ny, nz] at `iso` on the grid xs, ys, zs -> (verts [V, 3] float32, faces [F, 3] int64), on the
    device.  Inside is sigma > iso (NaN is outside); one vertex per grid edge that crosses the level, shared by its cells; face
    normals point toward decreasing density.  Deterministic; synchronises once to size the outputs."""
    sigma = _f32c(sigma, "sigma")
    if sigma.dim() != 3:
        raise RuntimeError(f"nerf_b200.marching_cubes: sigma must be [nx, ny, nz] (got shape {tuple(sigma.shape)})")
    dev = sigma.device
    xs, ys, zs = _axis(xs, "xs", dev), _axis(ys, "ys", dev), _axis(zs, "zs", dev)
    nx, ny, nz = sigma.shape
    if (xs.numel(), ys.numel(), zs.numel()) != (nx, ny, nz):
        raise RuntimeError(f"nerf_b200.marching_cubes: axes of {xs.numel()}, {ys.numel()}, {zs.numel()} points for sigma {tuple(sigma.shape)}")
    lib = _lib.load()
    ws_bytes = lib.nerf_b200_marching_cubes_workspace_bytes(nx, ny, nz)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    st = _stream(sigma)
    with _on(sigma):
        check(lib.nerf_b200_marching_cubes_count(_ptr(sigma), nx, ny, nz, float(iso), _ptr(counts), _ptr(ws), ws_bytes, st),
              "marching_cubes_count")
        V, F = (int(v) for v in counts.tolist())
        verts = torch.empty((V, 3), device=dev, dtype=torch.float32)
        faces = torch.empty((F, 3), device=dev, dtype=torch.int32)
        check(lib.nerf_b200_marching_cubes_emit(_ptr(sigma), _ptr(xs), _ptr(ys), _ptr(zs), nx, ny, nz, float(iso), _ptr(verts), V,
                                                _ptr(faces), F, _ptr(ws), ws_bytes, st), "marching_cubes_emit")
    return verts, faces.long()


def extract_mesh(network_fn, network_query_fn, xs, ys, zs, iso):
    """The mesh of `network_fn`'s density at level `iso` on the grid xs, ys, zs: density_grid, then marching_cubes.  Usually
    network_fn = render_kwargs_test['network_fine']."""
    return marching_cubes(density_grid(network_fn, network_query_fn, xs, ys, zs), xs, ys, zs, iso)


@torch.no_grad()
def density_gradient(network_fn, network_query_fn, pts):
    """(sigma [...], grad [..., 3]) of `network_fn` at pts [..., 3] (float32, on pts' device): sigma = run_network(pts)[..., 3] in
    fp32, the pre-ReLU density without noise, and grad = dsigma/dx through the network and the positional encoding.  Always the
    exact fp32 path, whatever set_precision says, so the same bits in every precision and on every run; any net the exact path
    serves.  `multires` is read from `network_query_fn` as density_grid reads it."""
    if not isinstance(network_fn, NeRF):
        raise RuntimeError("nerf_b200.density_gradient: network must be a nerf_b200.NeRF")
    pts = _f32c(pts, "pts")
    if pts.shape[-1] != 3:
        raise RuntimeError(f"nerf_b200.density_gradient: pts must be [..., 3] (got shape {tuple(pts.shape)})")
    mr = getattr(network_query_fn, "multires", None)
    if mr is None:
        mr = (network_fn.input_ch - 3) // 6
    P = pts.numel() // 3
    sigma = torch.empty(pts.shape[:-1], device=pts.device, dtype=torch.float32)
    grad = torch.empty(pts.shape, device=pts.device, dtype=torch.float32)
    if P == 0:
        return sigma, grad
    lib = _lib.load()
    n = network_fn.net_params()
    ws_bytes = lib.nerf_b200_density_gradient_workspace_bytes(P, C.byref(n))
    ws = _workspace(ws_bytes, pts.device)
    with _on(pts):
        _call(lib, "nerf_b200_density_gradient", _ptr(pts), P, C.byref(n), int(mr), _ptr(sigma), _ptr(grad), _ptr(ws), ws_bytes,
              _stream(pts))
    return sigma, grad


@torch.no_grad()
def vertex_attributes(network_fn, network_query_fn, verts):
    """(normals [V, 3], colors [V, 3]) of the mesh vertices verts [V, 3], for save_ply.  normals = -grad / |grad| of
    density_gradient (toward decreasing density, as marching_cubes winds its faces), 0 where |grad| is 0 or not finite.  colors
    = sigmoid(run_network(verts, viewdirs = -normals)[..., :3]) in the current set_precision: the view head looking at the
    surface head-on from outside; a vertex without a normal is seen along a zero view direction (as density_grid's points are),
    and a net without view directions takes none.  Usually network_fn = render_kwargs_test['network_fine']."""
    verts = _f32c(verts, "verts")
    if verts.dim() != 2 or verts.shape[1] != 3:
        raise RuntimeError(f"nerf_b200.vertex_attributes: verts must be [V, 3] (got shape {tuple(verts.shape)})")
    _, grad = density_gradient(network_fn, network_query_fn, verts)
    norm = grad.norm(dim=-1, keepdim=True)
    ok = torch.isfinite(norm) & (norm > 0)
    zero = torch.zeros_like(grad)
    look = torch.where(ok, grad / norm, zero)                         # the viewing ray's direction, -normal
    normals = torch.where(ok, -look, zero)
    raw = network_query_fn(verts[:, None], look if network_fn.use_viewdirs else None, network_fn)
    return normals, torch.sigmoid(raw[:, 0, :3])


def save_ply(path, verts, faces, normals=None, colors=None):
    """Write a triangle mesh (verts [V, 3], faces [F, 3]; tensors or arrays) as binary little-endian PLY, with optional
    per-vertex normals [V, 3] (float properties nx ny nz) and colors [V, 3] in [0, 1] (uchar red green blue, converted as
    to8b converts images)."""
    def host(a):
        return a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    v = np.ascontiguousarray(host(verts), dtype="<f4").reshape(-1, 3)
    f = host(faces).reshape(-1, 3)
    fields, props = [("p", "<f4", (3,))], "property float x\nproperty float y\nproperty float z\n"
    if normals is not None:
        fields.append(("n", "<f4", (3,)))
        props += "property float nx\nproperty float ny\nproperty float nz\n"
    if colors is not None:
        fields.append(("c", "u1", (3,)))
        props += "property uchar red\nproperty uchar green\nproperty uchar blue\n"
    vrec = np.empty(len(v), dtype=fields)
    vrec["p"] = v
    if normals is not None:
        vrec["n"] = host(normals).reshape(-1, 3)
    if colors is not None:
        vrec["c"] = to8b(host(colors).astype(np.float32).reshape(-1, 3))
    rec = np.empty(len(f), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    rec["n"] = 3
    rec["idx"] = f
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {len(v)}\n{props}"
              f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(rec.tobytes())
