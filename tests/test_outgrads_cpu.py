"""Gradients of every output of raw2outputs / render_rays, host side (no GPU needed).

  * oracle/outgrads.adjoint (the restatement of csrc/small_kernels.cuh: raw2outputs_bwd_kernel with all six seeds) against
    float64 autograd of the composite, seed by seed and combined, with and without white background and noise;
  * the same restatement against the reference's own dL/draw (tests/golden/outgrads.npz, oracle/gen_outgrads_golden.py);
  * the loss-scale rule reduces to max |dL/drgb_map| when rgb_map is the only seed;
  * the library exports the NerfOutGrads entry points, and rejects a backward without any seed before it launches anything.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden, rel_l2
from oracle import outgrads as OG
from oracle import tc_emul

SINGLE = [(k,) for k in OG.SEEDS]
COMBOS = SINGLE + [("acc_map", "disp_map"), ("rgb_map", "acc_map", "disp_map", "raw"), OG.SEEDS]


def _problem(seed, white_bkgd, noisy, N=12, S=40):
    g = torch.Generator().manual_seed(seed)
    raw = torch.randn(N, S, 4, generator=g, dtype=torch.float64) * 2
    raw[3, :, 3] = -1.0                                         # no density at all: acc = 0, disp NaN
    raw[3, 5, 3] = 1e-300                                       # density > 0 whose alpha rounds to 0: the NaN reaches this sample
    z = torch.sort(torch.rand(N, S, generator=g, dtype=torch.float64) * 4 + 2, -1).values
    d = torch.randn(N, 3, generator=g, dtype=torch.float64)
    noise = torch.rand(N, S, generator=g, dtype=torch.float64) * 0.7 if noisy else None
    if noisy:
        raw[3, :, 3] = -2.0                                     # stays <= 0 with the noise
    seeds = dict(rgb_map=torch.randn(N, 3, generator=g, dtype=torch.float64), disp_map=torch.randn(N, generator=g, dtype=torch.float64),
                 acc_map=torch.randn(N, generator=g, dtype=torch.float64), depth_map=torch.randn(N, generator=g, dtype=torch.float64),
                 weights=torch.randn(N, S, generator=g, dtype=torch.float64), raw=torch.randn(N, S, 4, generator=g, dtype=torch.float64))
    return raw, z, d, noise, seeds


def _autograd(raw, z, d, white_bkgd, noise, seeds):
    r = raw.clone().requires_grad_(True)
    out = OG.composite(r, z, d, white_bkgd, noise)
    loss = sum((out[k] * v).sum() for k, v in seeds.items() if k != "raw")
    if "raw" in seeds:
        loss = loss + (r * seeds["raw"]).sum()
    loss.backward()
    return r.grad


@pytest.mark.parametrize("noisy", [False, True])
@pytest.mark.parametrize("white_bkgd", [False, True])
@pytest.mark.parametrize("keys", COMBOS, ids=["+".join(k) for k in COMBOS])
def test_adjoint_matches_fp64_autograd(keys, white_bkgd, noisy):
    raw, z, d, noise, all_seeds = _problem(1, white_bkgd, noisy)
    seeds = {k: all_seeds[k] for k in keys}
    ref = _autograd(raw, z, d, white_bkgd, noise, seeds)
    got = OG.adjoint(raw, z, d, white_bkgd, seeds, noise)
    nan_ref, nan_got = torch.isnan(ref), torch.isnan(got)
    assert torch.equal(nan_ref, nan_got), (keys, nan_ref.sum(), nan_got.sum())
    if "disp_map" in keys and not noisy:
        # acc = 0: the disp gradient is NaN, but relu's gradient passes it only where the density is > 0
        assert bool(nan_ref[3, 5, 3]) and int(nan_ref.sum()) == 1
    m = ~nan_ref
    assert torch.allclose(got[m], ref[m], rtol=1e-9, atol=1e-12), (keys, (got[m] - ref[m]).abs().max())


def test_disp_has_no_gradient_below_the_clamp():
    """depth / acc < 1e-10: disp = 1e10 is the clamp constant and carries no gradient (torch.max's subgradient)."""
    raw, z, d, _, seeds = _problem(2, False, False, N=4)
    z = z * 1e-12                                               # depth / acc ~ 1e-12 < 1e-10 on every ray
    g = {"disp_map": seeds["disp_map"]}
    got = OG.adjoint(raw, z, d, False, g)
    ref = _autograd(raw, z, d, False, None, g)
    ok = ~torch.isnan(ref)
    assert torch.equal(got[ok], ref[ok]) and float(got[ok].abs().max()) == 0.0


@pytest.mark.parametrize("case", ["a", "b", "c"])
@pytest.mark.parametrize("loss", ["acc", "disp", "raw", "all"])
def test_adjoint_matches_reference_draw(case, loss):
    fx = load_golden("outgrads")
    wb = bool(fx[f"{case}_white_bkgd"])
    N = fx[f"{case}_rays"].shape[1]
    for i in (0, 1):
        raw = torch.from_numpy(fx[f"{case}_r2o{i}_raw"]).double()
        z = torch.from_numpy(fx[f"{case}_r2o{i}_z"]).double()
        d = torch.from_numpy(fx[f"{case}_r2o{i}_d"]).double()
        noise = torch.from_numpy(fx[f"{case}_r2o{i}_noise"]).double()
        p = f"{case}_{loss}_r2o{i}_"
        seeds = {k: torch.from_numpy(fx[p + "g_" + k]).double() for k in OG.SEEDS if p + "g_" + k in fx}
        if i == 1 and loss in ("raw", "all"):
            # the loss's own term on raw (the fine pass's raw is render()'s extras['raw'])
            S = z.shape[1]
            w = 1.0 if loss == "raw" else 1e-3
            g_raw = torch.zeros_like(raw)
            g_raw[..., 3] = w * (raw[..., 3] > 0).double() / (N * S)
            g_raw[..., :3] = w * 2.0 * raw[..., :3] / (N * S * 3)
            seeds["raw"] = g_raw
        got = OG.adjoint(raw, z, d, wb, seeds, noise).numpy()
        ref = fx[p + "draw"].astype(np.float64)
        assert np.array_equal(np.isnan(got), np.isnan(ref)), (case, loss, i)
        # relative to the reference's norm, with a floor for what is fp32 cancellation noise in the reference (e.g. an acc seed
        # on a saturated ray, acc = 1, whose exact gradient is ~0) or an fp32 acc that is exactly 0 where fp64's is not
        floor = 1e-6 * max((float(v.abs().max()) for v in seeds.values()), default=0.0) * np.sqrt(ref.size)
        err = np.linalg.norm(np.nan_to_num(got - ref))
        assert err <= 1e-4 * np.linalg.norm(np.nan_to_num(ref)) + floor, (case, loss, i, rel_l2(got, ref))


def test_loss_scale_rule_reduces_to_rgb_absmax():
    raw, z, d, noise, seeds = _problem(3, True, True)
    g = {"rgb_map": seeds["rgb_map"] * 1e-3}
    amax = OG.loss_scale_amax(raw, z, d, True, g, noise)
    assert amax == float(g["rgb_map"].abs().max())
    assert tc_emul.loss_scale(amax) == tc_emul.loss_scale(float(np.abs(g["rgb_map"].numpy()).max()))
    # an acc-only loss: g_rgb = 0, and the scale still comes from the seed that is there
    amax_acc = OG.loss_scale_amax(raw, z, d, True, {"acc_map": seeds["acc_map"]}, noise)
    assert amax_acc == float(seeds["acc_map"].abs().max()) and tc_emul.loss_scale(amax_acc) != 1.0


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from nerf_pytorch_b200 import _lib
    return _lib


NEW = ("nerf_b200_raw2outputs_bwd_outs", "nerf_b200_march_bwd_outs", "nerf_b200_march_bwd_tc_outs", "nerf_b200_render_rays_bwd_tc_outs")


def test_outs_entry_points_are_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "nerf_b200.h")).read()
    declared = set(re.findall(r"\b(nerf_b200_[a-z0-9_]+)\s*\(", hdr))
    so = ctypes.CDLL(os.path.join(ROOT, "nerf-pytorch_b200", "libnerf_b200.so"))
    for name in NEW:
        assert name in declared and name in lib.SIGNATURES and hasattr(so, name), name
    assert ctypes.sizeof(lib.NerfOutGrads) == 6 * 8
    assert lib.load().nerf_b200_abi_version() == 1


def test_a_pass_without_seeds_is_rejected(lib):
    """All-NULL NerfOutGrads: refused with a message during argument validation (nothing is launched or dereferenced)."""
    L = lib.load()
    fake = ctypes.c_void_p(256)
    rc = L.nerf_b200_raw2outputs_bwd_outs(fake, fake, fake, 3, None, 8, 16, 0, ctypes.byref(lib.NerfOutGrads()), fake, None)
    assert rc != 0 and b"no output gradient" in L.nerf_b200_last_error()
    net, cfg, gr = lib.NerfNetParams(), lib.NerfRenderCfg(), lib.NerfNetGrads()
    save = lib.NerfTrainSave(fake, 0, fake, 0)
    rc = L.nerf_b200_march_bwd_tc_outs(fake, fake, None, 8, 16, ctypes.byref(net), fake, ctypes.byref(cfg), fake, ctypes.byref(save),
                                       ctypes.byref(lib.NerfOutGrads()), ctypes.byref(gr), fake, 0, None)
    assert rc != 0 and b"no output gradient" in L.nerf_b200_last_error()
    rc = L.nerf_b200_march_bwd_outs(fake, fake, None, 8, 16, ctypes.byref(net), None, ctypes.byref(cfg),
                                    ctypes.byref(lib.NerfOutGrads()), ctypes.byref(gr), fake, 0, None)
    assert rc != 0 and b"no output gradient" in L.nerf_b200_last_error()
