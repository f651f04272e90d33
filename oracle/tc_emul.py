"""Quantisation-aware restatement of the tensor-core path  --  TEST INFRASTRUCTURE ONLY.

The fp16-operand / fp32-accumulate forward (csrc/fused_wg.cuh) and the loss-scaled fp16 backward (csrc/bwd_wg.cuh)
restated with stock torch ops on the CPU: every tensor the kernels round to fp16 is rounded here at the same place,
sums are taken in float64 (the kernels accumulate in fp32; the difference is O(1e-7)).  It is the oracle for the
tensor-core GRADIENTS: the reference's own fp32 autograd (tests/golden/lego_grads.npz) differs from any 10-bit-mantissa
evaluation by ReLU-mask flips (tools/bwd_precision_study.py), so stage-by-stage parity of the CUDA backward is checked
against this module, and end-to-end parity against the golden vectors with the documented budget.

Follows run_nerf_helpers.py:96-119 (NeRF.forward) and its autograd backward; run_nerf.py:262-305 via oracle/torch_ref.
"""
from __future__ import annotations

import numpy as np
import torch

from . import torch_ref as T


def f16(x: torch.Tensor) -> torch.Tensor:
    """Round to fp16 (saturating like cvt.rn.satfinite) and return as float64."""
    return x.clamp(-65504.0, 65504.0).to(torch.float16).to(torch.float64)


def loss_scale(amax: float) -> float:
    """csrc/train_common.cuh: loss_scale_from_absmax."""
    if not (amax > 0.0) or not np.isfinite(amax):
        return 1.0
    return float(2.0 ** np.floor(np.log2(np.float32(2048.0) / np.float32(amax))))


def input_ch(L: int) -> int:
    """run_nerf_helpers.py:48-63: 3 + 6 L columns; L = 0 is i_embed = -1 (the raw coordinates)."""
    return 3 + 6 * L


def encode16(pts: torch.Tensor, L: int):
    """gamma(p) rounded to fp16 -> (enc16 [M, 3 + 6L], enc64 [M, 64]: the encoding record, zero past column 3 + 6L)."""
    enc16 = f16(T.embed(pts.to(torch.float32), L).to(torch.float64))
    return enc16, torch.nn.functional.pad(enc16, (0, 64 - enc16.shape[1]))


def forward(sd: dict, pts: torch.Tensor, viewdirs_rows: torch.Tensor, D: int = 8, skip: int = 4, L: int = 10, Lv: int = 4):
    """pts [M,3], viewdirs_rows [M,3] (the ray's direction repeated per sample) -> dict of the tensors the kernel keeps.

    L / Lv: multires / multires_views (0: i_embed = -1); skip -1: none.  enc16 [M, 3 + 6L], enc64 [M, 64] (the encoding
    record), h16[l] [M,256] (post-ReLU, fp16-rounded), pre[l] (fp64 pre-activations), feat16, hv16, pre_v, raw [M,4]."""
    sd = {k: v.to(torch.float64) for k, v in sd.items()}
    w16 = {k: f16(v) for k, v in sd.items() if k.endswith("weight")}
    ic = input_ch(L)
    enc16, enc64 = encode16(pts, L)
    encv = T.embed(viewdirs_rows.to(torch.float32), Lv).to(torch.float64)
    out = {"enc16": enc16, "enc64": enc64, "h16": [], "pre": [], "encv": encv}
    h16 = None
    h32 = None
    for l in range(D):
        W = w16[f"pts_linears.{l}.weight"]
        b = sd[f"pts_linears.{l}.bias"]
        if l == 0:
            pre = enc16 @ W.t() + b
        elif l == skip + 1:
            pre = enc16 @ W[:, :ic].t() + h16 @ W[:, ic:].t() + b
        else:
            pre = h16 @ W.t() + b
        h32 = torch.relu(pre)
        h16 = f16(h32)
        out["pre"].append(pre)
        out["h16"].append(h16)
    sigma = h32 @ sd["alpha_linear.weight"].t() + sd["alpha_linear.bias"]          # fp32 head on the un-rounded activations
    feat = h16 @ w16["feature_linear.weight"].t() + sd["feature_linear.bias"]
    feat16 = f16(feat)
    Wv = sd["views_linears.0.weight"]
    vb = encv @ Wv[:, 256:].t() + sd["views_linears.0.bias"]                       # per-ray view bias, fp32 on CUDA cores
    pre_v = feat16 @ w16["views_linears.0.weight"][:, :256].t() + vb
    hv = torch.relu(pre_v)
    rgb = hv @ sd["rgb_linear.weight"].t() + sd["rgb_linear.bias"]
    out.update(feat16=feat16, pre_v=pre_v, hv16=f16(hv), raw=torch.cat([rgb, sigma], -1))
    return out


def composite_adjoint(raw: torch.Tensor, z: torch.Tensor, rays_d: torch.Tensor, g_rgb: torch.Tensor, white_bkgd: bool):
    """dL/draw [N,S,4] given dL/drgb_map [N,3] (autograd through the restated raw2outputs, float64)."""
    raw = raw.detach().to(torch.float64).requires_grad_(True)
    rgb_map, _, _, _ = T.composite(raw, z.to(torch.float64), rays_d.to(torch.float64), white_bkgd)
    (rgb_map * g_rgb.to(torch.float64)).sum().backward()
    return raw.grad


def backward(sd: dict, acts: dict, masks: dict, d_raw: torch.Tensor, scale: float, ray_of_row: torch.Tensor, n_rays: int,
             D: int = 8, skip: int = 4, L: int = 10):
    """The backward of csrc/bwd_wg.cuh given the forward's saved tensors (L: multires; the view encoding is acts['encv']).

    acts: enc16, h16[l], feat16, hv16, encv (per row);  masks: 'h'[l] [M,256] bool (pre-activation > 0), 'hv' [M,128];
    d_raw [M,4] fp64 (unscaled).  Returns (grads by state_dict key, stages) where stages holds the loss-scaled fp16
    tensors the kernels write: d_hv16, step[j] (j = 0: d_feat16, j >= 1: dA16 of pts layer D - j)."""
    sd = {k: v.to(torch.float64) for k, v in sd.items()}
    w16 = {k: f16(v) for k, v in sd.items() if k.endswith("weight")}
    ic = input_ch(L)
    d_rgb, d_sig = d_raw[:, :3].to(torch.float64), d_raw[:, 3:4].to(torch.float64)
    g = {}
    d_hv16 = f16((d_rgb * scale) @ sd["rgb_linear.weight"] * masks["hv"])
    stages = {"d_hv16": d_hv16, "step": []}
    d_feat16 = f16(d_hv16 @ w16["views_linears.0.weight"][:, :256])
    stages["step"].append(d_feat16)
    dA = f16((d_feat16 @ w16["feature_linear.weight"] + (d_sig * scale) * sd["alpha_linear.weight"]) * masks["h"][D - 1])
    stages["step"].append(dA)
    dAs = {D - 1: dA}
    for l in range(D - 1, 0, -1):
        W = w16[f"pts_linears.{l}.weight"]
        Wh = W[:, ic:] if l == skip + 1 else W
        dA = f16((dAs[l] @ Wh) * masks["h"][l - 1])
        dAs[l - 1] = dA
        stages["step"].append(dA)
    inv = 1.0 / scale
    # weight gradients: fp16 operands, wide accumulation
    g["rgb_linear.weight"] = d_rgb.t() @ acts["hv16"]
    g["rgb_linear.bias"] = d_rgb.sum(0)
    g["alpha_linear.weight"] = d_sig.t() @ acts["h16"][D - 1]
    g["alpha_linear.bias"] = d_sig.sum(0)
    gv = torch.zeros_like(sd["views_linears.0.weight"])
    # feature_linear's output is not recorded: d_hv^T feat = (d_hv^T h_{D-1}) W_feat^T + (sum_rows d_hv) b_feat^T  (csrc/bwd_wg.cuh)
    gv[:, :256] = (d_hv16.t() @ acts["h16"][D - 1] * inv) @ sd["feature_linear.weight"].t() + torch.outer(d_hv16.sum(0) * inv, sd["feature_linear.bias"])
    dsum = torch.zeros((n_rays, 128), dtype=torch.float64).index_add_(0, ray_of_row, d_hv16 * inv)
    encv_ray = torch.zeros((n_rays, acts["encv"].shape[1]), dtype=torch.float64)
    encv_ray[ray_of_row] = acts["encv"]
    gv[:, 256:] = dsum.t() @ encv_ray
    g["views_linears.0.weight"] = gv
    g["views_linears.0.bias"] = d_hv16.sum(0) * inv
    g["feature_linear.weight"] = d_feat16.t() @ acts["h16"][D - 1] * inv
    g["feature_linear.bias"] = d_feat16.sum(0) * inv
    for l in range(D - 1, -1, -1):
        dA = dAs[l]
        if l == 0:
            gw = dA.t() @ acts["enc16"][:, :ic] * inv
        elif l == skip + 1:
            gw = torch.cat([dA.t() @ acts["enc16"][:, :ic], dA.t() @ acts["h16"][l - 1]], 1) * inv
        else:
            gw = dA.t() @ acts["h16"][l - 1] * inv
        g[f"pts_linears.{l}.weight"] = gw
        g[f"pts_linears.{l}.bias"] = dA.sum(0) * inv
    return g, stages
