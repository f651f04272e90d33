"""Why precision tc_split uses fp16 halves with a per-layer weight scale: the split-operand forward restated on the CPU
(tests/split_emul.py) on the trained fixtures, against the reference's golden outputs, at the gates the exact fp32 path meets
on an H100 (test_gpu_parity._check_trained_gates, fp32 branch) and the north-star rgb_map <= 1e-4.

Measured with this restatement (lego: 1024 rays; fern: its first 1024 rays):
                      rgb_map  acc_map  rgb0     acc0     w_coarse w_fine   z_fine
  fp16 halves, scaled lego  3.1e-7   5.5e-7   5.4e-8   6.3e-8   2.6e-7   1.8e-5   3.2e-6
                      fern  2.6e-5   1.3e-5   1.0e-7   7.2e-8
  bf16 halves         lego  1.8e-5   4.6e-5   6.8e-7   9.1e-7   5.7e-6   5.3e-4   2.7e-5   (w_fine misses 5e-4)
  one fp16 MMA        lego  5.1e-4   1.8e-3   5.2e-5   8.3e-5   4.6e-4   3.5e-2   4.0e-4   (tc_fp16)
The fine pass's deviations are knot flips of the resampling (a coarse weight moving a sample across a cdf knot), so they are
gated with room; the coarse pass's are the arithmetic's own."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2

import split_emul as E

GATES = {"rgb0": 2e-5, "acc0": 2e-5, "rgb_map": 1e-4, "acc_map": 1e-4, "w_coarse": 1e-5, "w_fine": 5e-4, "z_fine": 1e-4}


def _run(name, half, n):
    from oracle import nerf_oracle as O
    from oracle import synth
    fx = load_golden(name)
    w = load_golden("trained_weights")
    sc = {k[2:]: torch.from_numpy(v) for k, v in w.items() if k.startswith("c.")}
    sf = {k[2:]: torch.from_numpy(v) for k, v in w.items() if k.startswith("f.")}
    lego = name.startswith("trained_lego")
    sb = synth.ray_batch("lego" if lego else "fern", int(fx["N"]), seed=int(fx["ray_seed"]))
    packed = O.pack_rays(sb["H"], sb["W"], sb["K"], sb["rays"][0], sb["rays"][1], not lego, 2.0 if lego else 0.0, 6.0 if lego else 1.0, True)
    with torch.no_grad():
        o = E.render_rays(torch.from_numpy(packed.astype(np.float32))[:n], sc, sf, half, white_bkgd=lego)
    return {k: rel_l2(o[k].numpy(), fx[k][:n]) for k in GATES if k in fx}


@pytest.mark.parametrize("name", ["trained_lego_1024", "fern_ndc_4096"])
def test_fp16_halves_with_a_weight_scale_meet_the_fp32_gates(name):
    st = _run(name, "fp16", 1024)
    print(name, st)
    for k, v in st.items():
        assert v < GATES[k], (k, st)
    if "w_coarse" in st:                                      # the coarse pass is the arithmetic's own: far under its gate
        assert st["rgb0"] < 1e-6 and st["w_coarse"] < 2e-6, st


def test_bf16_halves_miss_the_fine_weights_gate():
    st = _run("trained_lego_1024", "bf16", 1024)
    print(st)
    assert st["rgb_map"] < GATES["rgb_map"] and st["w_fine"] > GATES["w_fine"], st


def test_one_fp16_mma_misses_the_north_star():
    st = _run("trained_lego_1024", None, 1024)
    assert st["rgb_map"] > 2 * GATES["rgb_map"], st
