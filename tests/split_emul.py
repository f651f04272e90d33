"""Split-operand restatement of the `tc_split` forward (csrc/fused_wg.cuh, march_split_kernel) on the CPU.

Every operand x of a tensor-core product is carried as two halves of a narrow type, x = hi + lo with hi = round(x) and
lo = round(x - hi), and each layer accumulates  bias + sum_k (hi_a hi_b + hi_a lo_b + lo_a hi_b)  in fp32: three MMAs per
K-step into one accumulator, the lo_a lo_b term dropped.  Activations are rounded to fp32 where the kernel holds them in
fp32 (the accumulator), the heads and the per-ray view bias are fp32 FMA chains on the un-split values, and sums are taken
in float64 (the kernel's fp32 accumulation differs by O(1e-7)).  `half` picks the narrow type:

- "fp16" (the kernel's choice): 11-bit halves, 22 bits together.  fp16's 5-bit exponent puts lo of a weight of ~0.06 near
  2^-15, among the subnormals, so each layer's weights are scaled by a power of two that brings the largest |w| into
  [2^13, 2^14) (split_scale_kernel); the accumulator is scaled back exactly.  Activations are not scaled;
- "bf16": fp32's exponent and no scale, but 8-bit halves, 16 bits together; tests/test_split_precision_cpu.py shows the
  fine pass's weights missing the fp32 gate with them.

It also carries the one-operand fp16 forward (`half` = None: one MMA, fp16 operands, as `tc_fp16`) for comparison.  The
pipeline around the network is oracle/torch_ref.py's (render_rays: linspace z, composite, det resampling, sort).
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import torch_ref as T


def _round(x: torch.Tensor, half: str) -> torch.Tensor:
    dt = torch.bfloat16 if half == "bf16" else torch.float16
    return x.to(dt).to(torch.float64)


def f32(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).to(torch.float64)


def split(x: torch.Tensor, half: str):
    """x (values representable in fp32) -> (hi, lo): hi = round(x), lo = round(x - hi); x - hi is exact in fp32."""
    hi = _round(x, half)
    return hi, _round(x - hi, half)


def weight_scale(w: torch.Tensor, half) -> float:
    """csrc/fused_tc.cuh split_scale_kernel: 2^(14 - e) with max|w| < 2^e (fp16 halves), else 1"""
    amax = float(w.abs().max())
    if half != "fp16" or amax == 0.0:
        return 1.0
    return float(2.0 ** (14 - np.frexp(np.float32(amax))[1]))


def linear(a: torch.Tensor, w: torch.Tensor, half, scale: float = 1.0) -> torch.Tensor:
    """a [M, K] @ w[N, K]^T as the kernel's MMAs: split halves of a and of w * scale (three products), divided by the scale;
    or one fp16 product (half None)."""
    if half is None:
        return _round(a, "fp16") @ _round(w, "fp16").t()
    ah, al = split(a, half)
    wh, wl = split(w * scale, half)
    return (ah @ wh.t() + ah @ wl.t() + al @ wh.t()) / scale


def mlp(sd: dict, x: torch.Tensor, half, ic: int = 63, icv: int = 27, skip: int = 4, D: int = 8) -> torch.Tensor:
    """torch_ref.mlp's network ([M, ic + icv] fp32 encodings -> [M, 4] rgb, sigma) with the tensor-core layers emulated."""
    sd = {k: v.to(torch.float64) for k, v in sd.items()}
    x = x.to(torch.float64)
    pts, views = x[:, :ic], x[:, ic:ic + icv]
    h = None
    for i in range(D):
        W, b = sd[f"pts_linears.{i}.weight"], sd[f"pts_linears.{i}.bias"]
        sc = weight_scale(W, half)
        if i == 0:
            pre = linear(pts, W, half, sc)
        elif i == skip + 1:
            pre = linear(pts, W[:, :ic], half, sc) + linear(h, W[:, ic:], half, sc)
        else:
            pre = linear(h, W, half, sc)
        h = torch.relu(f32(pre + b))
    if "output_linear.weight" in sd:
        return (h @ sd["output_linear.weight"].t() + sd["output_linear.bias"])[:, :4]
    sigma = h @ sd["alpha_linear.weight"].t() + sd["alpha_linear.bias"]
    Wf = sd["feature_linear.weight"]
    feat = f32(linear(h, Wf, half, weight_scale(Wf, half)) + sd["feature_linear.bias"])
    Wv = sd["views_linears.0.weight"]
    vb = f32(views @ Wv[:, 256:].t() + sd["views_linears.0.bias"])
    hv = torch.relu(f32(linear(feat, Wv[:, :256], half, weight_scale(Wv[:, :256], half)) + vb))
    rgb = hv @ sd["rgb_linear.weight"].t() + sd["rgb_linear.bias"]
    return torch.cat([rgb, sigma], -1)


def _query(sd: dict, pts: torch.Tensor, viewdirs: torch.Tensor, half, chunk: int = 32768) -> torch.Tensor:
    N, S, _ = pts.shape
    flat = T.embed(pts.reshape(-1, 3).to(torch.float32), 10)                   # per-octave sin / cos in fp32
    dirs = T.embed(viewdirs[:, None].expand(N, S, 3).reshape(-1, 3).to(torch.float32), 4)
    x = torch.cat([flat, dirs], -1)
    out = torch.cat([mlp(sd, x[i:i + chunk], half) for i in range(0, x.shape[0], chunk)], 0)
    return out.to(torch.float32).reshape(N, S, 4)


def render_rays(packed: torch.Tensor, sd_c: dict, sd_f: dict, half, S: int = 64, n_imp: int = 128, white_bkgd: bool = True) -> dict:
    """torch_ref.render_rays (perturb 0, no noise; packed [N, 11] fp32) with the emulated network on both passes."""
    o, d, near, far, vd = packed[:, 0:3], packed[:, 3:6], packed[:, 6:7], packed[:, 7:8], packed[:, 8:11]
    t = torch.linspace(0.0, 1.0, S)
    z = near * (1.0 - t) + far * t
    raw = _query(sd_c, o[:, None] + d[:, None] * z[..., None], vd, half)
    rgb0, disp0, acc0, w = T.composite(raw, z, d, white_bkgd)
    mid = 0.5 * (z[:, 1:] + z[:, :-1])
    zs = T.resample(mid, w[:, 1:-1], n_imp)
    zf, _ = torch.sort(torch.cat([z, zs], -1), -1)
    raw_f = _query(sd_f, o[:, None] + d[:, None] * zf[..., None], vd, half)
    rgb, disp, acc, wf = T.composite(raw_f, zf, d, white_bkgd)
    return {"rgb_map": rgb, "disp_map": disp, "acc_map": acc, "rgb0": rgb0, "disp0": disp0, "acc0": acc0,
            "w_coarse": w, "w_fine": wf, "z_fine": zf}
