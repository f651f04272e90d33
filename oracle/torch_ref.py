"""Plain-PyTorch restatement of the reference's (unfused) render path  --  TEST INFRASTRUCTURE ONLY.

Why it exists: BASELINE.json's target is ">= 10x the reference PyTorch-GPU rays/sec".  /root/reference
does not exist on the GPU box, so the stock scripts cannot be timed there.  This module states the same
op chain with stock torch ops at the reference's granularity (per-frequency sin/cos + cat, one addmm +
relu per layer, cat at the skip, 65 536-row network chunks, cumprod compositing, searchsorted/gather
resampling) so that `tools/torch_gpu_reference.py` can time "what the reference does on this GPU".
Nothing in the product imports it.  Pinned by tests/test_oracle_golden.py against the same
reference-generated vectors as the numpy oracle.

Citations are to /root/reference (run_nerf.py = R, run_nerf_helpers.py = H).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def embed(x: torch.Tensor, L: int) -> torch.Tensor:
    """H:24-45 -- x, then sin/cos of 2^k x for k < L, concatenated on the channel axis."""
    parts = [x]
    for k in range(L):
        parts += [torch.sin(x * 2.0 ** k), torch.cos(x * 2.0 ** k)]
    return torch.cat(parts, -1)


def mlp(sd: dict, x: torch.Tensor, ic: int = 63, icv: int = 27, skip: int = 4, D: int = 8) -> torch.Tensor:
    """H:96-119 with the reference's state_dict keys; x [M, ic + icv] -> [M, 4] (rgb, sigma).  skip -1: none.  A net without
    view directions (an output_linear head, H:117) returns the first four of its outputs, the ones raw2outputs reads."""
    pts, views = x[:, :ic], x[:, ic:ic + icv]
    h = pts
    for i in range(D):
        h = F.relu(F.linear(h, sd[f"pts_linears.{i}.weight"], sd[f"pts_linears.{i}.bias"]))
        if i == skip:
            h = torch.cat([pts, h], -1)
    if "output_linear.weight" in sd:
        return F.linear(h, sd["output_linear.weight"], sd["output_linear.bias"])[:, :4]
    sigma = F.linear(h, sd["alpha_linear.weight"], sd["alpha_linear.bias"])
    feat = F.linear(h, sd["feature_linear.weight"], sd["feature_linear.bias"])
    hv = F.relu(F.linear(torch.cat([feat, views], -1), sd["views_linears.0.weight"], sd["views_linears.0.bias"]))
    rgb = F.linear(hv, sd["rgb_linear.weight"], sd["rgb_linear.bias"])
    return torch.cat([rgb, sigma], -1)


def query(sd: dict, pts: torch.Tensor, viewdirs: torch.Tensor, netchunk: int = 65536) -> torch.Tensor:
    """R:37-51 (+ batchify R:27-34): [N,S,3], [N,3] -> [N,S,4]."""
    N, S, _ = pts.shape
    flat = embed(pts.reshape(-1, 3), 10)
    dirs = embed(viewdirs[:, None].expand(N, S, 3).reshape(-1, 3), 4)
    x = torch.cat([flat, dirs], -1)
    out = torch.cat([mlp(sd, x[i:i + netchunk]) for i in range(0, x.shape[0], netchunk)], 0)
    return out.reshape(N, S, 4)


def composite(raw: torch.Tensor, z: torch.Tensor, rays_d: torch.Tensor, white_bkgd: bool):
    """R:262-305 without noise."""
    dists = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], -1) * rays_d.norm(dim=-1, keepdim=True)
    rgb = torch.sigmoid(raw[..., :3])
    alpha = 1.0 - torch.exp(-F.relu(raw[..., 3]) * dists)
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    w = alpha * trans
    rgb_map = (w[..., None] * rgb).sum(-2)
    depth = (w * z).sum(-1)
    acc = w.sum(-1)
    disp = 1.0 / torch.max(1e-10 * torch.ones_like(depth), depth / acc)
    if white_bkgd:
        rgb_map = rgb_map + (1.0 - acc[:, None])
    return rgb_map, disp, acc, w


def resample(bins: torch.Tensor, w: torch.Tensor, n: int) -> torch.Tensor:
    """H:196-239, det=True."""
    w = w + 1e-5
    cdf = torch.cumsum(w / w.sum(-1, keepdim=True), -1)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
    u = torch.linspace(0.0, 1.0, n, device=bins.device).expand(bins.shape[0], n).contiguous()
    idx = torch.searchsorted(cdf, u, right=True)
    lo, hi = (idx - 1).clamp(min=0), idx.clamp(max=cdf.shape[-1] - 1)
    c0, c1 = torch.gather(cdf, 1, lo), torch.gather(cdf, 1, hi)
    b0, b1 = torch.gather(bins, 1, lo), torch.gather(bins, 1, hi)
    den = c1 - c0
    den = torch.where(den < 1e-5, torch.ones_like(den), den)
    return b0 + (u - c0) / den * (b1 - b0)


def render_rays(packed: torch.Tensor, sd_c: dict, sd_f: dict, S: int = 64, n_imp: int = 128, white_bkgd: bool = True) -> dict:
    """R:308-418, perturb = 0, no noise: packed [N,11] = o d near far viewdir."""
    o, d, near, far, vd = packed[:, 0:3], packed[:, 3:6], packed[:, 6:7], packed[:, 7:8], packed[:, 8:11]
    t = torch.linspace(0.0, 1.0, S, device=packed.device)
    z = near * (1.0 - t) + far * t
    raw = query(sd_c, o[:, None] + d[:, None] * z[..., None], vd)
    rgb0, disp0, acc0, w = composite(raw, z, d, white_bkgd)
    mid = 0.5 * (z[:, 1:] + z[:, :-1])
    zs = resample(mid, w[:, 1:-1], n_imp).detach()
    zf, _ = torch.sort(torch.cat([z, zs], -1), -1)
    raw = query(sd_f, o[:, None] + d[:, None] * zf[..., None], vd)
    rgb, disp, acc, _ = composite(raw, zf, d, white_bkgd)
    return {"rgb_map": rgb, "disp_map": disp, "acc_map": acc, "rgb0": rgb0, "disp0": disp0, "acc0": acc0,
            "z_std": zs.std(-1, unbiased=False), "raw": raw}


def render(rays_o: torch.Tensor, rays_d: torch.Tensor, sd_c: dict, sd_f: dict, near: float, far: float,
           chunk: int = 32768, **kw) -> dict:
    """R:69-134 (non-NDC, use_viewdirs): normalise view directions, pack, march in `chunk`-ray slices."""
    vd = rays_d / rays_d.norm(dim=-1, keepdim=True)
    packed = torch.cat([rays_o, rays_d, near * torch.ones_like(rays_d[:, :1]), far * torch.ones_like(rays_d[:, :1]), vd], -1)
    outs = [render_rays(packed[i:i + chunk], sd_c, sd_f, **kw) for i in range(0, packed.shape[0], chunk)]
    return {k: torch.cat([o_[k] for o_ in outs], 0) for k in outs[0]}
