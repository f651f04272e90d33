"""CPU checks of the no-view-direction training path (use_viewdirs=False, output_linear head): the quantisation-aware
restatement in oracle/noviews.py against the numpy oracle and against autograd of its own forward, and the static shape of
the new seed kernel in the sm_90a SASS (no GPU needed)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O
from oracle import noviews as NV


class _RoundSTE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return x.clamp(-65504.0, 65504.0).to(torch.float16).to(torch.float64)

    @staticmethod
    def backward(ctx, g):
        return g


def _pts(M, seed=0):
    return torch.from_numpy(np.random.default_rng(seed).uniform(-2, 2, (M, 3)).astype(np.float32))


@pytest.mark.parametrize("output_ch", [5, 4])
def test_forward_noviews_matches_the_oracle(output_ch):
    """fp16 operands / fp32 head vs the fp32 numpy restatement of run_network (run_nerf.py:37-51) without view directions:
    the difference is the fp16 class (operands rounded to 11 bits)."""
    state = NV.nerf_state_noviews(3, output_ch=output_ch)
    assert state["output_linear.weight"].shape == (output_ch, 256) and state["views_linears.0.weight"].shape == (128, 256)
    pts = _pts(4 * 48)
    em = NV.forward_noviews({k: torch.from_numpy(v) for k, v in state.items()}, pts)
    ref = O.run_network(pts.numpy().reshape(4, 48, 3), None, state).reshape(-1, output_ch)
    err = float(np.linalg.norm(em["raw"].numpy() - ref[:, :4]) / np.linalg.norm(ref[:, :4]))
    assert err < 5e-3, err
    assert len(em["h16"]) == 8 and em["enc16"].shape == (4 * 48, 63)


def test_backward_noviews_is_the_gradient_of_the_emulated_forward():
    """The hand-written backward equals autograd of the forward with every fp16 rounding a straight-through estimator, up to the
    rounding of the activation gradients themselves; rows >= 4 of output_linear get no gradient."""
    rng = np.random.default_rng(1)
    M, D, skip, ic = 96, 8, 4, 63
    pts = _pts(M, 2)
    state = NV.nerf_state_noviews(4, sharpen=True)
    sd = {k: torch.from_numpy(v) for k, v in state.items()}
    em = NV.forward_noviews(sd, pts)
    r = _RoundSTE.apply
    sd_g = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    from oracle import torch_ref as T
    enc16 = r(T.embed(pts.float(), 10).double())
    h16 = None
    for l in range(D):
        W, b = r(sd_g[f"pts_linears.{l}.weight"]), sd_g[f"pts_linears.{l}.bias"]
        pre = enc16 @ W.t() + b if l == 0 else (enc16 @ W[:, :ic].t() + h16 @ W[:, ic:].t() + b if l == skip + 1 else h16 @ W.t() + b)
        h32 = torch.relu(pre)
        h16 = r(h32)
    raw = h32 @ sd_g["output_linear.weight"][:4].t() + sd_g["output_linear.bias"][:4]
    assert torch.allclose(raw, em["raw"], rtol=1e-9, atol=1e-9)
    d_raw = torch.from_numpy(rng.standard_normal((M, 4))).double() * 1e-3
    (raw * d_raw).sum().backward()
    masks = {"h": [(p > 0).double() for p in em["pre"]]}
    g, st = NV.backward_noviews(sd, em, masks, d_raw, 2.0 ** 16)
    assert len(st["step"]) == D + 1 and st["step"][0] is None
    for name, ref in sd_g.items():
        a = g[name].reshape(-1)
        b = ref.grad.reshape(-1) if ref.grad is not None else torch.zeros_like(a)
        if float(b.norm()) == 0.0:
            assert float(a.abs().max()) == 0.0, name
            continue
        err = float((a - b).norm() / b.norm())
        assert err < 2e-3, (name, err)
    assert float(g["output_linear.weight"][4].abs().max()) == 0.0 and float(g["output_linear.bias"][4]) == 0.0


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    ge.build()
    from nerf_pytorch_b200 import _lib
    return _lib.LIB_PATH


def test_seed_kernel_in_sass_without_local_memory(built):
    """dA_seed_output_kernel (bwd_wg.cuh) is compiled for sm_90a, keeps everything in registers (stack 0, no STL/LDL) and writes
    saturating fp16 (F2FP.SATFINITE)."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    usage = subprocess.run([exe, "-res-usage", built], capture_output=True, text=True, timeout=600).stdout.splitlines()
    found = [(ln, usage[i + 1]) for i, ln in enumerate(usage[:-1]) if re.search(r"Function \S*dA_seed_output_kernel\S*:", ln)]
    assert len(found) == 1, found
    m = re.search(r"REG:(\d+) STACK:(\d+)", found[0][1])
    assert m and int(m.group(2)) == 0, found
    sass = subprocess.run([exe, "-sass", built], capture_output=True, text=True, timeout=600).stdout
    bodies, cur = {}, None
    for ln in sass.splitlines():
        mm = re.search(r"Function : (\S+)", ln)
        if mm:
            cur = mm.group(1); bodies[cur] = []
        elif cur is not None:
            bodies[cur].append(ln)
    names = [k for k in bodies if "dA_seed_output_kernel" in k]
    assert len(names) == 1, names
    body = "\n".join(bodies[names[0]])
    assert not re.search(r"\b(STL|LDL)\b", body)
    assert "F2FP.SATFINITE" in body
