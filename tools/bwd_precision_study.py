"""CPU study for the round-2 tensor-core backward: which operand format may the gradient GEMMs use?

Emulates the planned dataflow of one network pass on the CPU (numpy): forward with fp16 weights / activations and fp32
accumulation (what march_wg_kernel does), then dgrad  dH = dA W  and wgrad  dW = dA^T H  with the activation-gradient
operand dA rounded to a candidate format (weights and saved activations stay fp16, accumulation fp32), and compares
every parameter gradient with a float64 evaluation of the exact algorithm (oracle.nerf_backward).

    python tools/bwd_precision_study.py [n_rays]

Formats: fp32 (no rounding: isolates the effect of the fp16 forward), tf32 (10-bit mantissa, fp32 range: what the
reference itself runs with under torch 1.11's allow_tf32 default), bf16, fp16 (raw: underflows), fp16 with one
power-of-two loss scale per tensor, fp16 with ONE static scale 2^floor(log2(3N * 1024)) derived from the batch size
(|dL/drgb| <= 2/(3N)), fp16 with a power-of-two scale per 128-row tile.
"""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import nerf_oracle as O, synth


def rnd_bits(x, keep):
    """round-to-nearest-even an fp32 array to `keep` explicit mantissa bits (tf32: 10, bf16: 7)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    drop = 23 - keep
    u = u + ((1 << (drop - 1)) - 1) + ((u >> drop) & 1)
    return ((u >> drop) << drop).astype(np.uint32).view(np.float32)


def q_fp16(x):
    with np.errstate(over="ignore"):
        return x.astype(np.float16).astype(np.float32)


def pow2_scale(amax, target=2.0 ** 12):
    return np.where(amax > 0, 2.0 ** np.floor(np.log2(np.maximum(target / np.maximum(amax, 1e-300), 1e-300))), 1.0)


STATIC_N = 1


def quant(x, fmt):
    if fmt == "fp32": return x
    if fmt == "tf32": return rnd_bits(x, 10)
    if fmt == "bf16": return rnd_bits(x, 7)
    if fmt == "fp16": return q_fp16(x)
    if fmt == "fp16*pass":
        s = np.float32(pow2_scale(np.abs(x).max()))
        return q_fp16(x * s) / s
    if fmt == "fp16*static":                        # one compile-time-like scale from the batch size: |dL/drgb| <= 2/(3N)
        s = np.float32(2.0 ** np.floor(np.log2(3.0 * STATIC_N * 1024.0)))
        return q_fp16(x * s) / s
    if fmt == "fp16*tile":
        M = x.shape[0]
        pad = (-M) % 128
        xp = np.concatenate([x, np.zeros((pad, x.shape[1]), x.dtype)]) if pad else x
        t = xp.reshape(-1, 128, x.shape[1])
        s = pow2_scale(np.abs(t).max(axis=(1, 2), keepdims=True)).astype(np.float32)
        return (q_fp16(t * s) / s).reshape(-1, x.shape[1])[:M]
    raise ValueError(fmt)


def backward_emulated(p, x, dout, ic, icv, fmt, skips=(4,), fwd="fp16"):
    """oracle.nerf_backward with the tensor-core operand roundings (run_nerf_helpers.py:96-119 in reverse).
    fwd = "fp16": this repo's forward operands; "tf32": what torch's matmul does under allow_tf32 (the reference's
    default with its pinned torch 1.11)."""
    f16 = (lambda a: q_fp16(np.asarray(a, np.float32))) if fwd == "fp16" else (lambda a: rnd_bits(np.asarray(a, np.float32), 10))
    W = {k: (f16(v) if k.endswith("weight") and not k.startswith(("alpha", "rgb")) else v.astype(np.float32)) for k, v in p.items()}
    pts, views = f16(x[:, :ic]), x[:, ic:ic + icv].astype(np.float32)
    D = 8
    ins, pre = [], []
    h = pts
    for i in range(D):
        ins.append(h)
        a = h @ W[f"pts_linears.{i}.weight"].T + W[f"pts_linears.{i}.bias"]
        pre.append(a)
        h = f16(np.maximum(a, 0))                       # the next layer's A operand is fp16
        if i in skips:
            h = np.concatenate([pts, h], -1)
    h_last = h
    feat = f16(h_last @ W["feature_linear.weight"].T + W["feature_linear.bias"])
    wv = W["views_linears.0.weight"]
    hv_pre = feat @ wv[:, :256].T + views @ p["views_linears.0.weight"][:, 256:].T.astype(np.float32) + W["views_linears.0.bias"]
    hv = np.maximum(hv_pre, 0)                          # rgb head runs in fp32 on CUDA cores
    g = {}
    d_rgb, d_alpha = dout[:, :3].astype(np.float32), dout[:, 3:4].astype(np.float32)
    g["rgb_linear.weight"] = d_rgb.T @ hv
    g["rgb_linear.bias"] = d_rgb.sum(0)
    d_hv = (d_rgb @ W["rgb_linear.weight"]) * (hv_pre > 0)              # K = 3: CUDA cores, fp32
    qd = quant(d_hv, fmt)
    g["views_linears.0.weight"] = np.concatenate([qd.T @ feat, d_hv.T @ views], -1)   # view columns: fp32 side path
    g["views_linears.0.bias"] = d_hv.sum(0)
    d_feat = qd @ wv[:, :256]
    qd = quant(d_feat, fmt)
    g["feature_linear.weight"] = qd.T @ h_last
    g["feature_linear.bias"] = d_feat.sum(0)
    g["alpha_linear.weight"] = d_alpha.T @ h_last
    g["alpha_linear.bias"] = d_alpha.sum(0)
    dh = qd @ W["feature_linear.weight"] + d_alpha @ W["alpha_linear.weight"]
    for i in reversed(range(D)):
        if i in skips:
            dh = dh[:, ic:]
        da = dh * (pre[i] > 0)
        qd = quant(da, fmt)
        g[f"pts_linears.{i}.weight"] = qd.T @ ins[i]
        g[f"pts_linears.{i}.bias"] = da.sum(0)
        if i > 0:
            dh = qd @ W[f"pts_linears.{i}.weight"]
    return g


def main():
    global STATIC_N
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 96
    STATIC_N = n
    sb = synth.ray_batch("lego", n, seed=3)
    packed = O.pack_rays(sb["H"], sb["W"], sb["K"], sb["rays"][0], sb["rays"][1], False, 2.0, 6.0, True)
    target = np.random.default_rng(1).random((n, 3)).astype(np.float32)
    for sharpen in (False, True):
        pc, pf = synth.nerf_state(0, sharpen), synth.nerf_state(1, sharpen)
        r = O.render_rays(packed, pc, 64, p_fine=pf, N_importance=128, retraw=True, white_bkgd=True, return_debug=True)
        z, raw = r["_debug"]["z_vals"], r["raw"]
        g_rgb = (2.0 * (r["rgb_map"] - target) / (3 * n)).astype(np.float32)
        draw = O.raw2outputs_backward(raw, z, packed[:, 3:6], g_rgb, True).reshape(-1, 4)
        pts = packed[:, None, 0:3] + packed[:, None, 3:6] * z[:, :, None]
        x = np.concatenate([O.embed(pts.reshape(-1, 3), 10), O.embed(np.broadcast_to(packed[:, None, 8:11], pts.shape).reshape(-1, 3), 4)], -1)
        ref = O.nerf_backward({k: v.astype(np.float64) for k, v in pf.items()}, x.astype(np.float64), draw.astype(np.float64), 63, 27)
        print(f"--- fine pass, {n} rays x 192 samples, sharpen={sharpen}: |dL/draw| max {np.abs(draw).max():.2e}, "
              f"median nonzero {np.median(np.abs(draw[draw != 0])):.2e}")
        print(f"{'format':10s} {'median rel-L2':>14s} {'max rel-L2':>12s}  worst tensor")
        for fmt in ("fp32", "tf32", "bf16", "fp16", "fp16*pass", "fp16*static", "fp16*tile"):
            g = backward_emulated(pf, x, draw, 63, 27, fmt)
            errs = sorted((float(np.linalg.norm(g[k] - ref[k]) / max(np.linalg.norm(ref[k]), 1e-300)), k) for k in ref)
            print(f"{fmt:10s} {np.median([e for e, _ in errs]):14.2e} {errs[-1][0]:12.2e}  {errs[-1][1]}")
        g = backward_emulated(pf, x, draw, 63, 27, "tf32", fwd="tf32")
        errs = sorted((float(np.linalg.norm(g[k] - ref[k]) / max(np.linalg.norm(ref[k]), 1e-300)), k) for k in ref)
        print(f"{'(all-TF32 matmuls, the reference GPU default)':46s} median {np.median([e for e, _ in errs]):.2e}  max {errs[-1][0]:.2e}  {errs[-1][1]}")


if __name__ == "__main__":
    main()
