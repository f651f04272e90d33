"""CPU oracle for the NeRF ray-marching hot path  --  TEST INFRASTRUCTURE ONLY.

This file is a plain-numpy restatement of the algorithm of yenchenlin/nerf-pytorch's
`render -> render_rays -> run_network -> NeRF.forward -> raw2outputs (+ sample_pdf)` path.
It is the *checker* for the CUDA product in `nerf-pytorch_b200/`; nothing in the product
imports it.  Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import this module.

Parity status: PINNED.  `oracle/gen_golden.py` imports the unmodified reference from
/root/reference (CPU, torch 2.11) and stores its inputs/outputs under `tests/golden/`;
`tests/test_oracle_golden.py` checks every function below against those vectors and against
the known-answer values recorded in SURVEY.md Appendix D.

Every function cites the reference file:line it follows (paths relative to /root/reference).
All arithmetic is done in `dtype` (float32 by default, like the reference; float64 available
to judge which of two fp32 implementations is closer to the truth).
"""
from __future__ import annotations

import numpy as np

from oracle import resample

# --------------------------------------------------------------------------------------
# Positional encoding  (run_nerf_helpers.py:15-63)
# --------------------------------------------------------------------------------------

def embed(x: np.ndarray, num_freqs: int) -> np.ndarray:
    """[..., 3] -> [..., 3 + 6*num_freqs]; order x, sin(2^0 x), cos(2^0 x), sin(2^1 x), ...

    run_nerf_helpers.py:24-45 (include_input, log_sampling: freqs = 2**linspace(0, L-1, L),
    which are exact powers of two), periodic_fns = [sin, cos] (:58).
    """
    out = [x]
    for k in range(num_freqs):
        f = x.dtype.type(2.0 ** k)
        out.append(np.sin(x * f))
        out.append(np.cos(x * f))
    return np.concatenate(out, -1)


def embed_out_dim(num_freqs: int, i_embed: int = 0) -> int:
    """run_nerf_helpers.py:48-63: i_embed == -1 -> identity (3 channels)."""
    return 3 if i_embed == -1 else 3 + 6 * num_freqs


# --------------------------------------------------------------------------------------
# NeRF MLP  (run_nerf_helpers.py:67-119)
# --------------------------------------------------------------------------------------

def _linear(x, w, b):
    return x @ w.T + b


def nerf_forward(p: dict, x: np.ndarray, input_ch: int, input_ch_views: int,
                 skips=(4,), use_viewdirs=True, return_hidden=False):
    """x [M, input_ch + input_ch_views] -> [M, 4].  `p` uses the reference's state_dict keys.

    run_nerf_helpers.py:96-119.  Skip: h = cat([input_pts, h]) AFTER layer i in skips (:102-103);
    alpha from h (:106), feature (:107), cat([feature, views]) (:108), relu(views_linears[0])
    (:110-112), rgb (:114), out = cat([rgb, alpha]) (:115).
    """
    input_pts, input_views = x[:, :input_ch], x[:, input_ch:input_ch + input_ch_views]
    h = input_pts
    D = len([k for k in p if k.startswith("pts_linears.") and k.endswith(".weight")])
    hidden = []
    for i in range(D):
        h = _linear(h, p[f"pts_linears.{i}.weight"], p[f"pts_linears.{i}.bias"])
        h = np.maximum(h, 0)
        hidden.append(h)
        if i in skips:
            h = np.concatenate([input_pts, h], -1)
    if use_viewdirs:
        alpha = _linear(h, p["alpha_linear.weight"], p["alpha_linear.bias"])
        feature = _linear(h, p["feature_linear.weight"], p["feature_linear.bias"])
        hv = np.concatenate([feature, input_views], -1)
        hv = np.maximum(_linear(hv, p["views_linears.0.weight"], p["views_linears.0.bias"]), 0)
        rgb = _linear(hv, p["rgb_linear.weight"], p["rgb_linear.bias"])
        out = np.concatenate([rgb, alpha], -1)
        if return_hidden:
            return out, hidden, feature, hv
        return out
    out = _linear(h, p["output_linear.weight"], p["output_linear.bias"])
    if return_hidden:
        return out, hidden, None, None
    return out


def run_network(inputs, viewdirs, p, multires=10, multires_views=4, i_embed=0,
                skips=(4,), netchunk=1024 * 64):
    """inputs [N,S,3], viewdirs [N,3] or None -> raw [N,S,C].  run_nerf.py:37-51 (+ batchify :27-34)."""
    N, S = inputs.shape[:2]
    flat = inputs.reshape(-1, 3)
    emb = embed(flat, multires) if i_embed != -1 else flat
    input_ch = emb.shape[-1]
    input_ch_views = 0
    if viewdirs is not None:
        dirs = np.broadcast_to(viewdirs[:, None], inputs.shape).reshape(-1, 3)   # :44-45
        emb_d = embed(dirs, multires_views) if i_embed != -1 else dirs
        input_ch_views = emb_d.shape[-1]
        emb = np.concatenate([emb, emb_d], -1)                                   # :47
    outs = []
    for i in range(0, emb.shape[0], netchunk):                                   # :27-34
        outs.append(nerf_forward(p, emb[i:i + netchunk], input_ch, input_ch_views,
                                 skips=skips, use_viewdirs=viewdirs is not None))
    out = np.concatenate(outs, 0)
    return out.reshape(N, S, out.shape[-1])


# --------------------------------------------------------------------------------------
# raw2outputs  (run_nerf.py:262-305)
# --------------------------------------------------------------------------------------

def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def raw2outputs(raw, z_vals, rays_d, noise=None, white_bkgd=False):
    """raw [N,S,>=4], z_vals [N,S], rays_d [N,3] -> rgb_map, disp_map, acc_map, weights, depth_map.

    run_nerf.py:277-303.  `noise` ([N,S] already scaled by raw_noise_std) replaces the
    reference's RNG draw (:285 / pytest :290) so that parity does not depend on an RNG stream.
    """
    dt = raw.dtype.type
    dists = z_vals[..., 1:] - z_vals[..., :-1]                                   # :277
    dists = np.concatenate([dists, np.full_like(dists[..., :1], 1e10)], -1)      # :278
    dists = dists * np.linalg.norm(rays_d[..., None, :], axis=-1).astype(raw.dtype)  # :280
    rgb = _sigmoid(raw[..., :3])                                                 # :282
    sigma = raw[..., 3] if noise is None else raw[..., 3] + noise                # :293
    with np.errstate(over="ignore"):
        alpha = dt(1.0) - np.exp(-np.maximum(sigma, 0) * dists)                  # :275
    ones = np.ones((alpha.shape[0], 1), raw.dtype)
    trans = np.cumprod(np.concatenate([ones, dt(1.0) - alpha + dt(1e-10)], -1), -1)[:, :-1]
    weights = alpha * trans                                                      # :295
    rgb_map = np.sum(weights[..., None] * rgb, -2)                               # :296
    depth_map = np.sum(weights * z_vals, -1)                                     # :298
    acc_map = np.sum(weights, -1)                                                # :300
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = depth_map / acc_map
        # torch.max(a, b) propagates NaN (SURVEY 8c); np.maximum does too.
        disp_map = dt(1.0) / np.maximum(dt(1e-10), ratio)                        # :299
    if white_bkgd:
        rgb_map = rgb_map + (dt(1.0) - acc_map[..., None])                       # :302-303
    return rgb_map, disp_map, acc_map, weights, depth_map


# --------------------------------------------------------------------------------------
# sample_pdf  (run_nerf_helpers.py:196-239)
# --------------------------------------------------------------------------------------

def sample_pdf(bins, weights, N_samples, det=False, u=None, pytest=False):
    """bins [N,B], weights [N,B-1] -> samples [N,N_samples].

    run_nerf_helpers.py:198-237, rounded as the reference on CPU torch (oracle/resample.py).  `u`
    ([N,N_samples]) replaces the RNG draw (:208 / :216); det without `u` takes torch.linspace (:205), or
    np.linspace under `pytest` (:215).  searchsorted(right=True) (:223) == first index with cdf > u.
    """
    return resample.sample_pdf(bins, weights, N_samples, det, u, pytest, dtype=bins.dtype)


# --------------------------------------------------------------------------------------
# z sampling + render_rays  (run_nerf.py:308-418)
# --------------------------------------------------------------------------------------

def coarse_z_vals(near, far, N_samples, lindisp=False, perturb=0.0, t_rand=None):
    """near, far [N,1] -> z_vals [N,N_samples].  run_nerf.py:357-379."""
    if perturb > 0.0:
        assert t_rand is not None, "stratified jitter must be injected"
    return resample.coarse_z(near, far, N_samples, lindisp, t_rand if perturb > 0.0 else None, dtype=near.dtype)


def render_rays(ray_batch, p_coarse, N_samples, p_fine=None, N_importance=0, retraw=False,
                lindisp=False, perturb=0.0, white_bkgd=False, t_rand=None, u=None,
                noise0=None, noise1=None, multires=10, multires_views=4, i_embed=0,
                return_debug=False):
    """ray_batch [N, 8|11] -> dict like the reference's render_rays (run_nerf.py:351-412).

    RNG draws are injected: t_rand [N,N_samples] (:371), u [N,N_importance] (sample_pdf :208),
    noise0/noise1 [N,S] sigma noise already scaled by raw_noise_std (:285).
    """
    N = ray_batch.shape[0]
    rays_o, rays_d = ray_batch[:, 0:3], ray_batch[:, 3:6]                        # :351
    viewdirs = ray_batch[:, -3:] if ray_batch.shape[-1] > 8 else None            # :352
    near, far = ray_batch[:, 6:7], ray_batch[:, 7:8]                             # :353-354
    z_vals = coarse_z_vals(near, far, N_samples, lindisp, perturb, t_rand)
    pts = rays_o[:, None, :] + rays_d[:, None, :] * z_vals[:, :, None]           # :381
    raw = run_network(pts, viewdirs, p_coarse, multires, multires_views, i_embed)  # :385
    rgb_map, disp_map, acc_map, weights, depth_map = raw2outputs(raw, z_vals, rays_d, noise0, white_bkgd)
    dbg = {"z_vals0": z_vals, "weights0": weights, "raw0": raw, "depth0": depth_map}
    if N_importance > 0:
        rgb0, disp0, acc0 = rgb_map, disp_map, acc_map                           # :390
        z_mid = z_vals.dtype.type(0.5) * (z_vals[..., 1:] + z_vals[..., :-1])    # :392
        z_samples = sample_pdf(z_mid, weights[..., 1:-1], N_importance,
                               det=(perturb == 0.0), u=u)                        # :393
        z_vals = np.sort(np.concatenate([z_vals, z_samples], -1), -1)            # :396
        pts = rays_o[:, None, :] + rays_d[:, None, :] * z_vals[:, :, None]       # :397
        run_p = p_coarse if p_fine is None else p_fine                           # :399
        raw = run_network(pts, viewdirs, run_p, multires, multires_views, i_embed)  # :401
        rgb_map, disp_map, acc_map, weights, depth_map = raw2outputs(raw, z_vals, rays_d, noise1, white_bkgd)
        dbg.update({"z_samples": z_samples})
    ret = {"rgb_map": rgb_map, "disp_map": disp_map, "acc_map": acc_map}         # :405
    if retraw:
        ret["raw"] = raw
    if N_importance > 0:
        ret["rgb0"], ret["disp0"], ret["acc0"] = rgb0, disp0, acc0               # :409-411
        ret["z_std"] = resample.z_std(z_samples)                                 # :412 (unbiased=False)
    if return_debug:
        dbg.update({"z_vals": z_vals, "weights": weights, "depth_map": depth_map})
        ret["_debug"] = dbg
    return ret


# --------------------------------------------------------------------------------------
# rays + render  (run_nerf_helpers.py:153-192, run_nerf.py:69-134)
# --------------------------------------------------------------------------------------

def get_rays_np(H, W, K, c2w, dtype=np.float32):
    """run_nerf_helpers.py:165-172."""
    i, j = np.meshgrid(np.arange(W, dtype=dtype), np.arange(H, dtype=dtype), indexing="xy")
    dirs = np.stack([(i - K[0][2]) / K[0][0], -(j - K[1][2]) / K[1][1], -np.ones_like(i)], -1)
    rays_d = np.sum(dirs[..., np.newaxis, :] * c2w[:3, :3], -1)
    rays_o = np.broadcast_to(c2w[:3, -1], rays_d.shape)
    return rays_o.astype(dtype), rays_d.astype(dtype)


def ndc_rays(H, W, focal, near, rays_o, rays_d):
    """run_nerf_helpers.py:175-192."""
    dt = rays_o.dtype.type
    t = -(dt(near) + rays_o[..., 2]) / rays_d[..., 2]
    rays_o = rays_o + t[..., None] * rays_d
    o0 = dt(-1.0 / (W / (2.0 * focal))) * rays_o[..., 0] / rays_o[..., 2]
    o1 = dt(-1.0 / (H / (2.0 * focal))) * rays_o[..., 1] / rays_o[..., 2]
    o2 = dt(1.0) + dt(2.0 * near) / rays_o[..., 2]
    d0 = dt(-1.0 / (W / (2.0 * focal))) * (rays_d[..., 0] / rays_d[..., 2] - rays_o[..., 0] / rays_o[..., 2])
    d1 = dt(-1.0 / (H / (2.0 * focal))) * (rays_d[..., 1] / rays_d[..., 2] - rays_o[..., 1] / rays_o[..., 2])
    d2 = dt(-2.0 * near) / rays_o[..., 2]
    return np.stack([o0, o1, o2], -1), np.stack([d0, d1, d2], -1)


def pack_rays(H, W, K, rays_o, rays_d, ndc, near, far, use_viewdirs):
    """The ray-batch construction inside render(): run_nerf.py:102-123 -> [N, 8|11]."""
    viewdirs = None
    if use_viewdirs:
        viewdirs = rays_d / np.linalg.norm(rays_d, axis=-1, keepdims=True)      # :108
        viewdirs = viewdirs.reshape(-1, 3).astype(np.float32)
    if ndc:
        rays_o, rays_d = ndc_rays(H, W, K[0][0], 1.0, rays_o, rays_d)            # :114
    rays_o = rays_o.reshape(-1, 3).astype(np.float32)
    rays_d = rays_d.reshape(-1, 3).astype(np.float32)
    nearv = near * np.ones_like(rays_d[..., :1])
    farv = far * np.ones_like(rays_d[..., :1])
    rays = np.concatenate([rays_o, rays_d, nearv, farv], -1)                     # :121
    if use_viewdirs:
        rays = np.concatenate([rays, viewdirs], -1)                              # :123
    return rays


def render(H, W, K, p_coarse, p_fine, chunk=1024 * 32, rays=None, c2w=None, ndc=True, near=0.0,
           far=1.0, use_viewdirs=False, **kw):
    """run_nerf.py:69-134 (c2w_staticcam omitted: visualisation-only special case)."""
    if c2w is not None:
        rays_o, rays_d = get_rays_np(H, W, K, c2w)                               # :97
    else:
        rays_o, rays_d = rays
    sh = rays_d.shape
    packed = pack_rays(H, W, K, rays_o, rays_d, ndc, near, far, use_viewdirs)
    per_ray = ("t_rand", "u", "noise0", "noise1")
    outs = {}
    for i in range(0, packed.shape[0], chunk):                                   # batchify_rays :54-66
        kws = {k: (v[i:i + chunk] if (k in per_ray and v is not None) else v) for k, v in kw.items()}
        r = render_rays(packed[i:i + chunk], p_coarse, p_fine=p_fine, **kws)
        for k, v in r.items():
            outs.setdefault(k, []).append(v)
    outs = {k: np.concatenate(v, 0) for k, v in outs.items() if k != "_debug"}
    for k in outs:
        outs[k] = outs[k].reshape(list(sh[:-1]) + list(outs[k].shape[1:]))       # :127-129
    k_extract = ["rgb_map", "disp_map", "acc_map"]
    return [outs[k] for k in k_extract] + [{k: v for k, v in outs.items() if k not in k_extract}]


# --------------------------------------------------------------------------------------
# Backward (hand-derived adjoint; SURVEY Appendix E).  Checked against reference autograd
# through the golden gradient fixtures.
# --------------------------------------------------------------------------------------

def raw2outputs_backward(raw, z_vals, rays_d, g_rgb, white_bkgd=False, noise=None):
    """dL/draw [N,S,4] given g_rgb = dL/drgb_map [N,3] (the only output the training loss reads,
    run_nerf.py:765-772).  Adjoint of run_nerf.py:277-303."""
    dt = raw.dtype.type
    dists = z_vals[..., 1:] - z_vals[..., :-1]
    dists = np.concatenate([dists, np.full_like(dists[..., :1], 1e10)], -1)
    dists = dists * np.linalg.norm(rays_d[..., None, :], axis=-1).astype(raw.dtype)
    c = _sigmoid(raw[..., :3])
    s = raw[..., 3] if noise is None else raw[..., 3] + noise
    with np.errstate(over="ignore"):
        one_m_alpha = np.exp(-np.maximum(s, 0) * dists)
    alpha = dt(1.0) - one_m_alpha
    q = dt(1.0) - alpha + dt(1e-10)
    ones = np.ones((alpha.shape[0], 1), raw.dtype)
    T = np.cumprod(np.concatenate([ones, q], -1), -1)[:, :-1]
    w = alpha * T
    cc = c - dt(1.0) if white_bkgd else c
    e = np.sum(g_rgb[:, None, :] * cc, -1)                                       # e_k
    we = w * e
    suffix = np.cumsum(we[:, ::-1], -1)[:, ::-1] - we                           # sum_{j>k} w_j e_j
    dalpha = T * e - suffix / q
    with np.errstate(over="ignore", invalid="ignore"):
        ds = np.where(s > 0, dalpha * dists * one_m_alpha, dt(0.0))
    draw = np.zeros_like(raw)
    draw[..., :3] = (w[..., None] * g_rgb[:, None, :]) * c * (dt(1.0) - c)
    draw[..., 3] = ds
    return draw


def nerf_backward(p: dict, x: np.ndarray, dout: np.ndarray, input_ch: int, input_ch_views: int,
                  skips=(4,)):
    """Gradients of all parameters of NeRF.forward (use_viewdirs=True) given dout [M,4].
    Mirrors run_nerf_helpers.py:96-119 in reverse.  No gradient w.r.t. x (SURVEY 3.5)."""
    input_pts, input_views = x[:, :input_ch], x[:, input_ch:input_ch + input_ch_views]
    D = len([k for k in p if k.startswith("pts_linears.") and k.endswith(".weight")])
    # forward with saved activations
    ins, pre = [], []
    h = input_pts
    for i in range(D):
        ins.append(h)
        a = _linear(h, p[f"pts_linears.{i}.weight"], p[f"pts_linears.{i}.bias"])
        pre.append(a)
        h = np.maximum(a, 0)
        if i in skips:
            h = np.concatenate([input_pts, h], -1)
    h_last = h
    feature = _linear(h_last, p["feature_linear.weight"], p["feature_linear.bias"])
    hv_in = np.concatenate([feature, input_views], -1)
    hv_pre = _linear(hv_in, p["views_linears.0.weight"], p["views_linears.0.bias"])
    hv = np.maximum(hv_pre, 0)
    g = {}
    d_rgb, d_alpha = dout[:, :3], dout[:, 3:4]
    g["rgb_linear.weight"] = d_rgb.T @ hv
    g["rgb_linear.bias"] = d_rgb.sum(0)
    d_hv = (d_rgb @ p["rgb_linear.weight"]) * (hv_pre > 0)
    g["views_linears.0.weight"] = d_hv.T @ hv_in
    g["views_linears.0.bias"] = d_hv.sum(0)
    d_feature = (d_hv @ p["views_linears.0.weight"])[:, :feature.shape[1]]
    g["feature_linear.weight"] = d_feature.T @ h_last
    g["feature_linear.bias"] = d_feature.sum(0)
    g["alpha_linear.weight"] = d_alpha.T @ h_last
    g["alpha_linear.bias"] = d_alpha.sum(0)
    dh = d_feature @ p["feature_linear.weight"] + d_alpha @ p["alpha_linear.weight"]
    for i in reversed(range(D)):
        if i in skips:
            dh = dh[:, input_ch:]                                   # drop the encoded-input segment
        da = dh * (pre[i] > 0)
        g[f"pts_linears.{i}.weight"] = da.T @ ins[i]
        g[f"pts_linears.{i}.bias"] = da.sum(0)
        if i > 0:
            dh = da @ p[f"pts_linears.{i}.weight"]
    return g


def render_rays_grads(ray_batch, p_coarse, p_fine, N_samples, N_importance, target,
                      lindisp=False, perturb=0.0, white_bkgd=False, t_rand=None, u=None,
                      multires=10, multires_views=4):
    """loss = mse(rgb_map, target) + mse(rgb0, target) (run_nerf.py:765-772) and dL/dtheta for
    both networks.  Returns (loss, grads_coarse, grads_fine)."""
    r = render_rays(ray_batch, p_coarse, N_samples, p_fine=p_fine, N_importance=N_importance,
                    retraw=True, lindisp=lindisp, perturb=perturb, white_bkgd=white_bkgd,
                    t_rand=t_rand, u=u, multires=multires, multires_views=multires_views,
                    return_debug=True)
    dbg = r["_debug"]
    N = ray_batch.shape[0]
    rays_o, rays_d, viewdirs = ray_batch[:, 0:3], ray_batch[:, 3:6], ray_batch[:, -3:]
    dt = ray_batch.dtype.type
    loss = np.mean((r["rgb_map"] - target) ** 2)
    out = []
    passes = [("rgb0" if N_importance > 0 else "rgb_map", dbg["z_vals0"], dbg["raw0"], p_coarse)]
    if N_importance > 0:
        loss = loss + np.mean((r["rgb0"] - target) ** 2)
        passes.append(("rgb_map", dbg["z_vals"], r["raw"], p_fine if p_fine is not None else p_coarse))
    for key, z, raw, p in passes:
        g_rgb = dt(2.0) * (r[key] - target) / dt(3 * N)
        draw = raw2outputs_backward(raw, z, rays_d, g_rgb, white_bkgd)
        pts = rays_o[:, None, :] + rays_d[:, None, :] * z[:, :, None]
        S = z.shape[1]
        x = np.concatenate([embed(pts.reshape(-1, 3), multires),
                            embed(np.broadcast_to(viewdirs[:, None], pts.shape).reshape(-1, 3), multires_views)], -1)
        out.append(nerf_backward(p, x, draw.reshape(N * S, 4), 3 + 6 * multires, 3 + 6 * multires_views))
    return loss, out[0], (out[1] if len(out) > 1 else None)
