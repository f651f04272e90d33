"""Networks without view directions (`use_viewdirs=False`, the default of run_nerf.py:467)  --  TEST INFRASTRUCTURE ONLY.

Such a NeRF ends in `output_linear` (run_nerf_helpers.py:91-92, :117) with output_ch = 5 when N_importance > 0 and 4
otherwise (run_nerf.py:187); only its first four rows reach raw2outputs.  This module holds

  * nerf_state_noviews: deterministic parameters keyed like that network's state_dict (synth.nerf_state's counterpart);
  * forward_noviews / backward_noviews: the quantisation-aware restatement (as oracle/tc_emul.py for the view-direction
    net) of the tensor-core training forward (csrc/fused_wg.cuh) and backward (csrc/bwd_wg.cuh: dA_seed_output_kernel,
    then the dgrad chain from dA_{D-1} and the layer-major weight gradient).
"""
from __future__ import annotations

import numpy as np
import torch

from . import synth
from . import tc_emul
from .tc_emul import f16


def nerf_state_noviews(seed=0, sharpen=False, output_ch=5, D=8, W=256, input_ch=63, skips=(4,)):
    """pts_linears and views_linears.0 (created but unused without view directions, input_ch_views = 0) as
    synth.nerf_state draws them, plus output_linear [output_ch, W] with nn.Linear's default init distribution.
    sharpen=True scales the head like SURVEY 8d(ii): sigma row * 30, its bias + 0.5, rgb rows * 5."""
    base = synth.nerf_state(seed, False, D=D, W=W, input_ch=input_ch, input_ch_views=0, skips=skips)
    p = {k: v for k, v in base.items() if k.startswith(("pts_linears.", "views_linears."))}
    rng = np.random.default_rng(2000 + seed)
    b = 1.0 / np.sqrt(W)
    w = rng.uniform(-b, b, (output_ch, W)).astype(np.float32)
    bias = rng.uniform(-b, b, (output_ch,)).astype(np.float32)
    if sharpen:
        w[:3] *= np.float32(5)
        w[3] *= np.float32(30)
        bias[3] += np.float32(0.5)
    p["output_linear.weight"], p["output_linear.bias"] = w, bias
    return p


def forward_noviews(sd: dict, pts: torch.Tensor, D: int = 8, skip: int = 4, L: int = 10):
    """pts [M,3] -> dict: enc16 [M, 3 + 6L], enc64 [M, 64] (as tc_emul.forward; L = 0: i_embed = -1), h16[l] [M,256] (post-ReLU, fp16-rounded), pre[l] (fp64 pre-activations), raw [M,4].

    The head is fp32 on the UN-rounded h_{D-1} (the kernel's FMA chains on the accumulators); the training-mode pass
    records h16[D-1] besides, for output_linear's weight gradient."""
    sd = {k: v.to(torch.float64) for k, v in sd.items()}
    w16 = {k: f16(v) for k, v in sd.items() if k.endswith("weight")}
    ic = tc_emul.input_ch(L)
    enc16, enc64 = tc_emul.encode16(pts, L)
    out = {"enc16": enc16, "enc64": enc64, "h16": [], "pre": []}
    h16 = h32 = None
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
    out["raw"] = h32 @ sd["output_linear.weight"][:4].t() + sd["output_linear.bias"][:4]
    return out


def backward_noviews(sd: dict, acts: dict, masks: dict, d_raw: torch.Tensor, scale: float, D: int = 8, skip: int = 4, L: int = 10):
    """The backward of csrc/bwd_wg.cuh for an output_linear head, given the forward's saved tensors.

    acts: enc16, h16[l] (per row);  masks: 'h'[l] [M,256] (pre-activation > 0);  d_raw [M,4] fp64 (unscaled).
    Returns (grads by state_dict key, stages): stages['step'][j] for j = 1..D is the loss-scaled fp16 image the kernels write
    at step j of the gradient record, dA16 of pts layer D - j (index 0 unused: None)."""
    sd = {k: v.to(torch.float64) for k, v in sd.items()}
    w16 = {k: f16(v) for k, v in sd.items() if k.endswith("weight")}
    ic = tc_emul.input_ch(L)
    d4 = d_raw[:, :4].to(torch.float64)
    Wout = sd["output_linear.weight"]
    # seed: fp32 head weights, the ReLU mask of layer D-1, one saturating fp16 rounding
    dA = f16((d4 * scale) @ Wout[:4] * masks["h"][D - 1])
    stages = {"step": [None, dA]}
    dAs = {D - 1: dA}
    for l in range(D - 1, 0, -1):
        W = w16[f"pts_linears.{l}.weight"]
        Wh = W[:, ic:] if l == skip + 1 else W
        dA = f16((dAs[l] @ Wh) * masks["h"][l - 1])
        dAs[l - 1] = dA
        stages["step"].append(dA)
    inv = 1.0 / scale
    g = {}
    gw = torch.zeros_like(Wout)
    gb = torch.zeros_like(sd["output_linear.bias"])
    gw[:4] = d4.t() @ acts["h16"][D - 1]            # rows >= 4 never reach the loss: zero
    gb[:4] = d4.sum(0)
    g["output_linear.weight"], g["output_linear.bias"] = gw, gb
    for l in range(D - 1, -1, -1):
        dA = dAs[l]
        if l == 0:
            gwl = dA.t() @ acts["enc16"][:, :ic] * inv
        elif l == skip + 1:
            gwl = torch.cat([dA.t() @ acts["enc16"][:, :ic], dA.t() @ acts["h16"][l - 1]], 1) * inv
        else:
            gwl = dA.t() @ acts["h16"][l - 1] * inv
        g[f"pts_linears.{l}.weight"] = gwl
        g[f"pts_linears.{l}.bias"] = dA.sum(0) * inv
    if "views_linears.0.weight" in sd:                 # created by the reference's NeRF but unused: zero gradient
        g["views_linears.0.weight"] = torch.zeros_like(sd["views_linears.0.weight"])
        g["views_linears.0.bias"] = torch.zeros_like(sd["views_linears.0.bias"])
    return g, stages
