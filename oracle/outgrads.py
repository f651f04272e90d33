"""Gradients of every output of raw2outputs (run_nerf.py:262-305)  --  TEST INFRASTRUCTURE ONLY.

A loss may read any of rgb_map, disp_map, acc_map, depth_map, weights and raw (depth / disparity supervision, a mask
loss on acc_map, a density regulariser on raw[..., 3]).  This module restates, in float64 torch:

  * composite:  the forward with noise and depth (oracle/torch_ref.composite plus R:283-291 noise and R:298 depth), the
    function the reference's autograd differentiates;
  * adjoint:    the hand-derived adjoint the CUDA kernel computes (csrc/small_kernels.cuh: raw2outputs_bwd_kernel) for
    any subset of the six seeds;
  * loss_scale_amax: the tensor-core backward's loss-scale input over those seeds (include/nerf_b200.h,
    nerf_b200_march_bwd_tc_outs), which with dL/drgb_map alone is max |dL/drgb_map|.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import torch_ref as T

SEEDS = ("rgb_map", "disp_map", "acc_map", "depth_map", "weights", "raw")
LOSSES = ("acc", "disp", "raw", "all")


def loss_of(name, rgb, disp, acc, ex, target, t_acc):
    """The losses of tests/golden/outgrads.npz on render()'s outputs (any torch device):
    L_acc = mse(acc, t_a) + mse(acc0, t_a);  L_disp = mean(disp) + mean(disp0);
    L_raw = mean(relu(raw[..., 3])) + mean(raw[..., :3]^2);  L_all = img2mse(rgb) + img2mse(rgb0) + L_acc + 0.1 L_disp + 1e-3 L_raw."""
    l_acc = torch.mean((acc - t_acc) ** 2) + torch.mean((ex["acc0"] - t_acc) ** 2)
    l_disp = torch.mean(disp) + torch.mean(ex["disp0"])
    raw = ex["raw"]
    l_raw = torch.mean(torch.relu(raw[..., 3])) + torch.mean(raw[..., :3] ** 2)
    if name == "acc":
        return l_acc
    if name == "disp":
        return l_disp
    if name == "raw":
        return l_raw
    l_rgb = torch.mean((rgb - target) ** 2) + torch.mean((ex["rgb0"] - target) ** 2)
    return l_rgb + l_acc + 0.1 * l_disp + 1e-3 * l_raw


def trained_states(path):
    """(coarse, fine) state dicts of tests/golden/trained_weights.npz"""
    import numpy as np
    w = np.load(path)
    return [{k[2:]: w[k] for k in w.files if k.startswith(t + ".")} for t in ("c", "f")]


def noviews_from_trained(trained, seed):
    """A net without view directions (output_ch 5) with the trained net's density: its pts_linears, and output_linear's sigma
    row = the trained alpha_linear (sigma reads only those), the other rows from oracle/noviews.nerf_state_noviews(seed).
    A random net's density is positive at the far end of most rays, so acc = 1 exactly there (the last interval is 1e10)
    and an acc loss has a gradient of pure rounding noise; the trained density is zero in empty space (acc spans 0..1)."""
    from . import noviews
    st = noviews.nerf_state_noviews(seed)
    st.update({k: v for k, v in trained.items() if k.startswith("pts_linears.")})
    st["output_linear.weight"] = st["output_linear.weight"].copy()
    st["output_linear.bias"] = st["output_linear.bias"].copy()
    st["output_linear.weight"][3] = trained["alpha_linear.weight"][0]
    st["output_linear.bias"][3] = trained["alpha_linear.bias"][0]
    return st


def composite(raw, z, rays_d, white_bkgd, noise=None):
    """R:262-305 -> dict(rgb_map, disp_map, acc_map, depth_map, weights).  noise [N,S] (the reference's pytest draw
    times raw_noise_std) or None."""
    if noise is None:
        rgb, disp, acc, w = T.composite(raw, z, rays_d, white_bkgd)
        return dict(rgb_map=rgb, disp_map=disp, acc_map=acc, depth_map=(w * z).sum(-1), weights=w)
    dists = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], -1) * rays_d.norm(dim=-1, keepdim=True)
    c = torch.sigmoid(raw[..., :3])
    alpha = 1.0 - torch.exp(-F.relu(raw[..., 3] + noise) * dists)
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    w = alpha * trans
    rgb = (w[..., None] * c).sum(-2)
    depth = (w * z).sum(-1)
    acc = w.sum(-1)
    disp = 1.0 / torch.max(1e-10 * torch.ones_like(depth), depth / acc)
    if white_bkgd:
        rgb = rgb + (1.0 - acc[:, None])
    return dict(rgb_map=rgb, disp_map=disp, acc_map=acc, depth_map=depth, weights=w)


def effective_seeds(raw, z, rays_d, white_bkgd, g, noise=None):
    """Per-ray acc and depth seeds with disp_map's chain rule folded in: disp = 1 / max(1e-10, depth / acc).
    torch.max's subgradient: none where depth/acc < 1e-10, half at equality, NaN where acc = 0 (ratio NaN)."""
    N = z.shape[0]
    zero = torch.zeros(N, dtype=z.dtype, device=z.device)
    g_acc = g["acc_map"].to(z.dtype).clone() if g.get("acc_map") is not None else zero.clone()
    g_depth = g["depth_map"].to(z.dtype).clone() if g.get("depth_map") is not None else zero.clone()
    if g.get("disp_map") is not None:
        with torch.no_grad():
            o = composite(raw, z, rays_d, white_bkgd, noise)
        depth, acc = o["depth_map"], o["acc_map"]
        ratio = depth / acc
        mx = torch.where(torch.isnan(ratio), ratio, torch.clamp(ratio, min=1e-10))
        g_ratio = -g["disp_map"].to(z.dtype) / (mx * mx)
        g_ratio = torch.where(ratio < 1e-10, torch.zeros_like(g_ratio), torch.where(ratio == 1e-10, 0.5 * g_ratio, g_ratio))
        g_depth = g_depth + g_ratio / acc
        g_acc = g_acc - g_ratio * depth / (acc * acc)
    return g_acc, g_depth


def adjoint(raw, z, rays_d, white_bkgd, g, noise=None):
    """dL/draw [N,S,4] for the seeds in `g` (keys of SEEDS; missing or None = that output is not on the loss)."""
    raw, z, rays_d = raw.to(torch.float64), z.to(torch.float64), rays_d.to(torch.float64)
    noise = None if noise is None else noise.to(torch.float64)
    N, S = z.shape
    dists = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], -1) * rays_d.norm(dim=-1, keepdim=True)
    s = raw[..., 3] + (noise if noise is not None else 0.0)
    oma = torch.exp(-torch.relu(s) * dists)
    alpha = 1.0 - oma
    q = 1.0 - alpha + 1e-10
    Tr = torch.cumprod(torch.cat([torch.ones_like(q[:, :1]), q], -1), -1)[:, :-1]
    w = alpha * Tr
    c = torch.sigmoid(raw[..., :3])
    e = torch.zeros_like(w)
    d = torch.zeros_like(raw)
    if g.get("rgb_map") is not None:
        gr = g["rgb_map"].to(torch.float64)
        off = 1.0 if white_bkgd else 0.0
        e = e + ((c - off) * gr[:, None, :]).sum(-1)
        d[..., :3] = w[..., None] * gr[:, None, :] * c * (1.0 - c)
    if g.get("acc_map") is not None or g.get("disp_map") is not None or g.get("depth_map") is not None:
        g_acc, g_depth = effective_seeds(raw, z, rays_d, white_bkgd, g, noise)
        e = e + g_acc[:, None] + g_depth[:, None] * z
    if g.get("weights") is not None:
        e = e + g["weights"].to(torch.float64)
    we = w * e
    suffix = torch.flip(torch.cumsum(torch.flip(we, [-1]), -1), [-1]) - we          # sum_{j>k} w_j e_j
    dalpha = Tr * e - suffix / q
    d[..., 3] = torch.where(s > 0, dalpha * dists * oma, torch.zeros_like(s))     # relu's gradient is a select (NaN stays out)
    if g.get("raw") is not None:
        d = d + g["raw"].to(torch.float64)
    return d


def loss_scale_amax(raw, z, rays_d, white_bkgd, g, noise=None):
    """max( |g_rgb|, |g_acc_eff|, |g_depth_eff * z_k|, |g_weights|, |g_raw| ) over the seeds given (float64; NaN if any is).
    Rays whose disp is NaN (acc = 0) under a disp seed are left out of the acc / depth terms."""
    raw, z, rays_d = raw.to(torch.float64), z.to(torch.float64), rays_d.to(torch.float64)
    noise = None if noise is None else noise.to(torch.float64)
    parts = []
    if g.get("rgb_map") is not None:
        parts.append(g["rgb_map"].to(torch.float64).reshape(-1))
    has_acc = g.get("acc_map") is not None or g.get("disp_map") is not None
    has_depth = g.get("depth_map") is not None or g.get("disp_map") is not None
    if has_acc or has_depth:
        g_acc, g_depth = effective_seeds(raw, z, rays_d, white_bkgd, g, noise)
        keep = torch.ones_like(g_acc, dtype=torch.bool)
        if g.get("disp_map") is not None:
            with torch.no_grad():
                o = composite(raw, z, rays_d, white_bkgd, noise)
            keep = ~torch.isnan(o["depth_map"] / o["acc_map"])
        if has_acc:
            parts.append(g_acc[keep])
        if has_depth:
            parts.append((g_depth[:, None] * z)[keep].reshape(-1))
    for k in ("weights", "raw"):
        if g.get(k) is not None:
            parts.append(g[k].to(torch.float64).reshape(-1))
    a = torch.cat(parts).abs()
    return float("nan") if bool(torch.isnan(a).any()) else float(a.max())
