"""Pin the numpy oracle (oracle/nerf_oracle.py) against the reference's own outputs
(tests/golden/*.npz, produced by oracle/gen_golden.py from the unmodified reference) and the
known-answer values of SURVEY.md Appendix D.  CPU only."""
import numpy as np
import pytest

from conftest import load_golden, rel_l2
from oracle import nerf_oracle as O
from oracle import synth

CASES = ["lego_det", "lego_sharp_det", "lego_perturb", "lego_coarse_only", "lego_lindisp",
         "fern_ndc_det", "fern_ndc_noise"]


def run_oracle_case(fx, dtype=np.float32, return_debug=False):
    pc = synth.nerf_state(int(fx["seed_w"]), bool(fx["sharpen"]))
    pf = synth.nerf_state(int(fx["seed_w"]) + 1, bool(fx["sharpen"])) if int(fx["N_importance"]) > 0 else None
    if dtype != np.float32:
        pc = {k: v.astype(dtype) for k, v in pc.items()}
        pf = {k: v.astype(dtype) for k, v in pf.items()} if pf else None
    rays = fx["rays"]
    packed = O.pack_rays(int(fx["H"]), int(fx["W"]), fx["K"], rays[0], rays[1], bool(fx["ndc"]),
                         float(fx["near"]), float(fx["far"]), True).astype(dtype)
    return O.render_rays(packed, pc, int(fx["N_samples"]), p_fine=pf, N_importance=int(fx["N_importance"]),
                         retraw=True, lindisp=bool(fx["lindisp"]), perturb=float(fx["perturb"]),
                         white_bkgd=bool(fx["white_bkgd"]), t_rand=fx.get("t_rand"), u=fx.get("u"),
                         noise0=fx.get("noise0"), noise1=fx.get("noise1"), return_debug=return_debug)


@pytest.mark.parametrize("name", CASES)
def test_render_matches_reference(name):
    fx = load_golden(name)
    r = run_oracle_case(fx)
    # fp32 restatement; only BLAS summation order and libm differ from the reference.  The
    # reference's own distance to an fp64 evaluation is of the same size (maps ~1e-7..1e-6,
    # fine-pass raw 2e-5..6e-4 because 2^9-frequency encodings amplify 1-ulp z differences).
    tol = {"rgb_map": 1e-5, "acc_map": 1e-5, "rgb0": 1e-5, "acc0": 1e-5, "z_std": 2e-5,
           "raw": 3e-3 if bool(fx["sharpen"]) else 2e-4}
    for k, t in tol.items():
        if k in fx:
            assert rel_l2(r[k], fx[k]) < t, (name, k, rel_l2(r[k], fx[k]))
    for k in ("disp_map", "disp0"):
        if k in fx:
            assert np.array_equal(np.isnan(r[k]), np.isnan(fx[k])), (name, k)
            assert rel_l2(r[k], fx[k]) < 1e-3, (name, k, rel_l2(r[k], fx[k]))


def test_units_embed():
    fx = load_golden("units")
    for L in (10, 4, 2):
        got = O.embed(fx["embed_x"], L)
        assert got.shape == fx[f"embed_L{L}"].shape
        np.testing.assert_allclose(got, fx[f"embed_L{L}"], atol=2e-6, rtol=0)


def test_units_nerf_forward():
    fx = load_golden("units")
    y = O.nerf_forward(synth.nerf_state(7), fx["nerf_x"], 63, 27)
    assert rel_l2(y, fx["nerf_y"]) < 5e-6


def test_units_raw2outputs():
    fx = load_golden("units")
    for tag, wb, noise in (("wb0", False, None), ("wb1", True, None), ("noise", True, fx["r2o_noise"])):
        outs = O.raw2outputs(fx["r2o_raw"], fx["r2o_z"], fx["r2o_d"], noise, wb)
        for nm, o in zip(("rgb", "disp", "acc", "weights", "depth"), outs):
            ref = fx[f"r2o_{nm}_{tag}"]
            assert np.array_equal(np.isnan(o), np.isnan(ref)), (tag, nm)
            np.testing.assert_allclose(np.nan_to_num(o), np.nan_to_num(ref), rtol=2e-5, atol=2e-6)
    assert np.isnan(fx["r2o_disp_wb0"][5])          # all sigma<=0 -> 0/0 (SURVEY App. D)


def test_units_sample_pdf():
    fx = load_golden("units")
    # The oracle rounds the sum, cumsum and linspace as CPU torch does (oracle/resample.py), so even a u
    # on a cdf knot (notably u == 1 vs cdf[-1], SURVEY App. D quirk 5) takes the reference's bin.
    det = O.sample_pdf(fx["spdf_bins"], fx["spdf_w"], 128, det=True)
    assert np.array_equal(det, fx["spdf_det"])
    rnd = O.sample_pdf(fx["spdf_bins"], fx["spdf_w"], 128, det=False, u=fx["spdf_u"])
    assert np.array_equal(rnd, fx["spdf_rand"])


def test_units_rays():
    fx = load_golden("units")
    o, d = O.get_rays_np(40, 40, fx["rays_K"], fx["rays_c2w"])
    np.testing.assert_allclose(o, fx["rays_o"], atol=1e-6)
    np.testing.assert_allclose(d, fx["rays_d"], atol=1e-6)
    c2wf = synth.fern_camera()[3]
    o, d = O.get_rays_np(38, 50, fx["ndc_K"], c2wf)
    no, nd = O.ndc_rays(38, 50, fx["ndc_K"][0][0], 1.0, o, d)
    np.testing.assert_allclose(no, fx["ndc_o"], atol=1e-6)
    np.testing.assert_allclose(nd, fx["ndc_d"], atol=1e-6)


def test_known_answers_appendix_d():
    """SURVEY.md Appendix D known-answer values recorded from the reference."""
    e = O.embed(np.array([[0.1, 0.2, 0.3]], np.float32), 2)[0]
    np.testing.assert_allclose(e, [0.1, 0.2, 0.3, 0.099833, 0.198669, 0.295520, 0.995004, 0.980067,
                                   0.955337, 0.198669, 0.389418, 0.564642, 0.980067, 0.921061, 0.825336], atol=1e-6)
    assert O.embed_out_dim(10) == 63 and O.embed_out_dim(4) == 27 and O.embed_out_dim(10, -1) == 3
    s = O.sample_pdf(np.array([[0, 1, 2, 3]], np.float32), np.array([[1, 2, 1]], np.float32), 5, det=True)[0]
    np.testing.assert_allclose(s, [0.0, 0.999997, 1.5, 2.000002, 3.0], atol=2e-6)
    s = O.sample_pdf(np.array([[0, 1, 2, 3]], np.float32), np.zeros((1, 3), np.float32), 5, det=True)[0]
    np.testing.assert_allclose(s, [0, 0.75, 1.5, 2.25, 3.0], atol=2e-6)
    np.random.seed(0)
    u = np.random.rand(1, 4).astype(np.float32)
    s = O.sample_pdf(np.array([[0, 1, 2, 3]], np.float32), np.array([[1, 2, 1]], np.float32), 4, u=u)[0]
    np.testing.assert_allclose(s, [1.597627, 1.930380, 1.705527, 1.589767], atol=2e-6)
    raw = np.array([[[0, 0, 0, -1], [1, -1, 0, .5], [0, 2, 0, 3], [0, 0, 0, -.1]]], np.float32)
    z = np.linspace(2, 6, 4, dtype=np.float32)[None]
    d = np.array([[0, 0, -2]], np.float32)
    rgb, disp, acc, w, depth = O.raw2outputs(raw, z, d)
    np.testing.assert_allclose(w[0], [0, 0.736403, 0.263509, 0], atol=1e-6)
    np.testing.assert_allclose(rgb[0], [0.670108, 0.430147, 0.499956], atol=1e-6)
    np.testing.assert_allclose([disp[0], acc[0], depth[0]], [0.271392, 0.999912, 3.684384], atol=2e-6)
    rgbw = O.raw2outputs(raw, z, d, white_bkgd=True)[0]
    np.testing.assert_allclose(rgbw[0], [0.670196, 0.430235, 0.500044], atol=1e-6)
    neg = raw.copy(); neg[..., 3] = -1
    rgb, disp, acc, w, depth = O.raw2outputs(neg, z, d, white_bkgd=True)
    assert np.allclose(rgb, 1.0) and np.isnan(disp[0]) and acc[0] == 0 and depth[0] == 0
    tiny = neg.copy(); tiny[0, :3, 3] = [0.0, 0.5, 3.0]; tiny[0, 3, 3] = 1e-9
    w = O.raw2outputs(tiny, z, d)[3]
    np.testing.assert_allclose(w[0, 3], 8.842503e-05, rtol=1e-4)
    assert list(np.searchsorted([0, .25, .75, 1], [0, .25, .5, 1], side="right")) == [1, 2, 2, 4]


@pytest.mark.parametrize("name", ["lego_grads", "lego_sharp_grads"])
def test_gradients_match_reference_autograd(name):
    fx = load_golden(name)
    pc = synth.nerf_state(int(fx["seed_w"]), bool(fx["sharpen"]))
    pf = synth.nerf_state(int(fx["seed_w"]) + 1, bool(fx["sharpen"]))
    rays = fx["rays"]
    packed = O.pack_rays(int(fx["H"]), int(fx["W"]), fx["K"], rays[0], rays[1], False, 2.0, 6.0, True)
    loss, gc, gf = O.render_rays_grads(packed, pc, pf, 64, 128, fx["target"], white_bkgd=True)
    assert abs(loss - fx["loss"]) / fx["loss"] < 1e-5
    worst = 0.0
    for tag, g in (("c", gc), ("f", gf)):
        for k, v in g.items():
            ref_norm = float(fx[f"g_{tag}_{k}_norm"])
            got_norm = float(np.linalg.norm(v.astype(np.float64)))
            assert abs(got_norm - ref_norm) <= (1e-3 if bool(fx["sharpen"]) else 5e-3) * ref_norm + 1e-9, (tag, k, got_norm, ref_norm)
            idx = fx[f"g_{tag}_{k}_idx"]
            err = np.linalg.norm(v.reshape(-1)[idx] - fx[f"g_{tag}_{k}_val"]) / max(np.linalg.norm(fx[f"g_{tag}_{k}_val"]), 1e-12)
            worst = max(worst, err)
            # sharpened heads amplify the MLP's fp32 summation order; the fine samples themselves are the
            # reference's (sample_pdf rounds like CPU torch).  Measured worst: 5.6e-3 sampled, 2e-4 on the norms.
            assert err < (1e-2 if bool(fx["sharpen"]) else 2e-3), (tag, k, err)


def test_fp64_oracle_is_consistent():
    fx = load_golden("lego_det")
    r32 = run_oracle_case(fx)
    r64 = run_oracle_case(fx, np.float64)
    assert rel_l2(r32["rgb_map"], r64["rgb_map"]) < 1e-5


@pytest.mark.parametrize("name", ["lego_det", "lego_sharp_det"])
def test_torch_restatement_matches_reference(name):
    """oracle/torch_ref.py (the op chain timed as the PyTorch-GPU baseline by tools/torch_gpu_reference.py)
    reproduces the reference's outputs on the deterministic lego fixtures."""
    import torch
    from oracle import torch_ref as T
    fx = load_golden(name)
    sd = [{k: torch.from_numpy(v) for k, v in synth.nerf_state(int(fx["seed_w"]) + i, bool(fx["sharpen"])).items()} for i in (0, 1)]
    rays = torch.from_numpy(fx["rays"])
    with torch.no_grad():
        r = T.render(rays[0], rays[1], sd[0], sd[1], float(fx["near"]), float(fx["far"]), S=int(fx["N_samples"]),
                     n_imp=int(fx["N_importance"]), white_bkgd=bool(fx["white_bkgd"]))
    for k, t in {"rgb_map": 1e-5, "acc_map": 1e-5, "rgb0": 1e-5, "acc0": 1e-5, "z_std": 2e-5}.items():
        assert rel_l2(r[k].numpy(), fx[k]) < t, (name, k, rel_l2(r[k].numpy(), fx[k]))
