"""GPU parity tests, kernel by kernel, through the C ABI (include/nerf_b200.h)."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


@pytest.mark.parametrize("K,N", [(32, 256), (64, 256), (256, 256), (256, 128), (128, 128)])
def test_wgmma_selftest_gemm(G, K, N):
    """Operand layouts (128B-swizzled A written by threads, 64B-swizzled weight chunks via bulk copy) and
    wgmma descriptors: D = fp16(A) fp16(W)^T with fp32 accumulation."""
    lib = G._lib.load_dev()
    rng = np.random.default_rng(K * 1000 + N)
    A = rng.standard_normal((128, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    a, w = G.dev(A), G.dev(W)
    out = torch.zeros((128, N), device=G.DEV)
    scratch = torch.zeros(N * K * 2, dtype=torch.uint8, device=G.DEV)
    G._lib.check_dev(lib.nerf_b200_selftest_gemm(G.ptr(a), G.ptr(w), K, N, G.ptr(out), G.ptr(scratch), scratch.numel(), G.stream()), "selftest")
    torch.cuda.synchronize()
    ref = A.astype(np.float16).astype(np.float64) @ W.astype(np.float16).astype(np.float64).T
    err = np.abs(out.cpu().numpy() - ref).max()
    assert err < 2e-3, err          # only fp32 accumulation order differs


def test_wgmma_selftest_gemm_tn(G):
    """MN-major operands straight from the activation layout (the weight-gradient GEMM's access pattern):
    out[256,256] = fp16(X)^T fp16(Y) over 128 sample rows, LBO = K-block stride, SBO = 8-row group stride."""
    lib = G._lib.load_dev()
    rng = np.random.default_rng(11)
    X = rng.standard_normal((128, 256)).astype(np.float32)
    Y = rng.standard_normal((128, 256)).astype(np.float32)
    x, y = G.dev(X), G.dev(Y)
    out = torch.zeros((256, 256), device=G.DEV)
    G._lib.check_dev(lib.nerf_b200_selftest_gemm_tn(G.ptr(x), G.ptr(y), G.ptr(out), 16384, 1024, G.stream()), "selftest_tn")
    torch.cuda.synchronize()
    ref = X.astype(np.float16).astype(np.float64).T @ Y.astype(np.float16).astype(np.float64)
    assert rel_l2(out.cpu().numpy(), ref) < 1e-5


def test_embed(G):
    fx = load_golden("units")
    for L in (10, 4, 2):
        fn, od = G.nb.get_embedder(L, 0)
        got = fn(G.dev(fx["embed_x"])).cpu().numpy()
        assert got.shape[-1] == od
        np.testing.assert_allclose(got, fx[f"embed_L{L}"], atol=2e-6, rtol=0)
    assert G.nb.get_embedder(10, -1)[1] == 3


def test_raw2outputs_forward(G):
    fx = load_golden("units")
    raw, z, d = G.dev(fx["r2o_raw"]), G.dev(fx["r2o_z"]), G.dev(fx["r2o_d"])
    for tag, wb in (("wb0", False), ("wb1", True)):
        outs = G.nb.raw2outputs(raw, z, d, 0, wb)
        for nm, o in zip(("rgb", "disp", "acc", "weights", "depth"), outs):
            ref = fx[f"r2o_{nm}_{tag}"]
            o = o.cpu().numpy()
            assert np.array_equal(np.isnan(o), np.isnan(ref)), (tag, nm)      # disp NaN when acc == 0
            np.testing.assert_allclose(np.nan_to_num(o), np.nan_to_num(ref), rtol=3e-5, atol=3e-6)
    outs = G.nb.raw2outputs(raw, z, d, 0.7, True, pytest=True)                 # pytest-hook noise (uniform)
    for nm, o in zip(("rgb", "disp", "acc", "weights", "depth"), outs):
        np.testing.assert_allclose(np.nan_to_num(o.cpu().numpy()), np.nan_to_num(fx[f"r2o_{nm}_noise"]), rtol=3e-5, atol=3e-6)


def test_raw2outputs_backward(G):
    rng = np.random.default_rng(11)
    raw = (rng.standard_normal((37, 45, 4)) * 1.5).astype(np.float32)
    z = np.sort(rng.random((37, 45), dtype=np.float32) * 4 + 2, -1)
    d = rng.standard_normal((37, 3)).astype(np.float32)
    g = rng.standard_normal((37, 3)).astype(np.float32)
    for wb in (False, True):
        t = G.dev(raw).requires_grad_(True)
        rgb = G.nb.raw2outputs(t, G.dev(z), G.dev(d), 0, wb)[0]
        rgb.backward(G.dev(g))
        ref = G.O.raw2outputs_backward(raw.astype(np.float64), z.astype(np.float64), d.astype(np.float64), g.astype(np.float64), wb)
        assert rel_l2(t.grad.cpu().numpy(), ref) < 2e-5


def test_sample_pdf(G):
    fx = load_golden("units")
    bins, w = G.dev(fx["spdf_bins"]), G.dev(fx["spdf_w"])
    det = G.nb.sample_pdf(bins, w, 128, det=True).cpu().numpy()
    rnd = G.nb.sample_pdf(bins, w, 128, det=False, pytest=True).cpu().numpy()
    for got, ref in ((det, fx["spdf_det"]), (rnd, fx["spdf_rand"])):
        np.testing.assert_array_equal(got, ref)      # the cdf rounds like CPU torch's (oracle/resample.py)


def test_coarse_z_and_fine_z(G):
    lib = G._lib.load()
    fx = load_golden("lego_perturb")
    rays = G.dev(G.packed_rays(fx))
    N = rays.shape[0]
    t_vals = torch.linspace(0., 1., 64, device=G.DEV)
    for lindisp in (0, 1):
        for t_rand in (None, G.dev(fx["t_rand"])):
            z = torch.empty((N, 64), device=G.DEV)
            G._lib.check(lib.nerf_b200_coarse_z(G.ptr(rays), 11, G.ptr(t_vals), G.ptr(t_rand), N, 64, lindisp, G.ptr(z), G.stream()), "coarse_z")
            near, far = G.packed_rays(fx)[:, 6:7], G.packed_rays(fx)[:, 7:8]
            ref = G.O.coarse_z_vals(near, far, 64, bool(lindisp), 1.0 if t_rand is not None else 0.0,
                                    fx["t_rand"] if t_rand is not None else None)
            np.testing.assert_array_equal(z.cpu().numpy(), ref)
    # fine_z == sort(cat[z, sample_pdf(mid, w[1:-1])]) and z_std
    rng = np.random.default_rng(5)
    zc = np.sort(rng.random((N, 64), dtype=np.float32) * 4 + 2, -1)
    w = rng.random((N, 64), dtype=np.float32) ** 3
    u = rng.random((N, 128), dtype=np.float32)
    zf = torch.empty((N, 192), device=G.DEV); zs = torch.empty((N, 128), device=G.DEV); zstd = torch.empty(N, device=G.DEV)
    d_zc, d_w, d_u = G.dev(zc), G.dev(w), G.dev(u)          # keep the inputs alive across the call
    G._lib.check(lib.nerf_b200_fine_z(G.ptr(d_zc), G.ptr(d_w), G.ptr(d_u), 128, N, 64, 128, G.ptr(zf), G.ptr(zs), G.ptr(zstd), G.stream()), "fine_z")
    torch.cuda.synchronize()
    mid = 0.5 * (zc[:, 1:] + zc[:, :-1])
    ref_s = G.O.sample_pdf(mid, w[:, 1:-1], 128, u=u)
    np.testing.assert_array_equal(zs.cpu().numpy(), ref_s)
    got = zf.cpu().numpy()
    assert np.all(np.diff(got, axis=-1) >= 0)                                   # sortedness
    np.testing.assert_array_equal(got, np.sort(np.concatenate([zc, zs.cpu().numpy()], -1), -1))   # a permutation of its inputs
    np.testing.assert_array_equal(zstd.cpu().numpy(), G.O.resample.z_std(ref_s))


@pytest.mark.parametrize("prec,tol", [("fp32", 2e-5), ("tc_fp16", 3e-3)])
def test_run_network(G, prec, tol):
    """encode + NeRF.forward: run_network(pts, viewdirs) vs the oracle (raw, before compositing)."""
    rng = np.random.default_rng(21)
    N, S = 37, 50                                   # ragged: 1850 rows, not a multiple of 128
    pts = (rng.random((N, S, 3), dtype=np.float32) * 6 - 3)
    vd = rng.standard_normal((N, 3)).astype(np.float32); vd /= np.linalg.norm(vd, axis=-1, keepdims=True)
    st = G.synth.nerf_state(7)
    net = G.make_net(st)
    q = G.query_fn()
    G.nb.set_precision(prec)
    try:
        got = q(G.dev(pts), G.dev(vd), net).cpu().numpy()
    finally:
        G.nb.set_precision("tc_fp16")
    ref = G.O.run_network(pts, vd, st)
    assert got.shape == ref.shape
    assert rel_l2(got, ref) < tol, rel_l2(got, ref)


def test_run_network_no_viewdirs(G):
    rng = np.random.default_rng(22)
    N, S = 16, 64
    pts = (rng.random((N, S, 3), dtype=np.float32) * 4 - 2)
    st = G.synth.nerf_state(9)
    st = {k: v for k, v in st.items() if k.startswith("pts_linears")}
    b = 1.0 / 16.0
    st["output_linear.weight"] = rng.uniform(-b, b, (5, 256)).astype(np.float32)
    st["output_linear.bias"] = rng.uniform(-b, b, (5,)).astype(np.float32)
    st["views_linears.0.weight"] = rng.uniform(-b, b, (128, 256)).astype(np.float32)   # present in the module, unused
    st["views_linears.0.bias"] = rng.uniform(-b, b, (128,)).astype(np.float32)
    net = G.make_net(st, use_viewdirs=False, output_ch=5)
    e, _ = G.nb.get_embedder(10, 0)
    q = G._QueryFn(e, None, 65536, 10, 4, 0)
    for prec, tol in (("fp32", 2e-5), ("tc_fp16", 3e-3)):
        G.nb.set_precision(prec)
        try:
            got = q(G.dev(pts), None, net).cpu().numpy()
        finally:
            G.nb.set_precision("tc_fp16")
        ref = G.O.run_network(pts, None, st)[..., :4]
        assert rel_l2(got, ref) < tol, (prec, rel_l2(got, ref))


def test_pack_rays_matches_reference_ray_construction(G):
    """get_rays + viewdir normalisation + ndc_rays + packing (run_nerf.py:95-123) vs golden reference rays and the oracle."""
    import ctypes as C
    fx = load_golden("units")
    lib = G._lib.load()
    # 1. generated lego rays (no NDC) == reference get_rays
    from nerf_pytorch_b200.api import _camera
    cam = _camera(40, 40, fx["rays_K"], fx["rays_c2w"])
    out = torch.empty((1600, 11), device=G.DEV)
    G._lib.check(lib.nerf_b200_pack_rays(None, None, None, C.byref(cam), 1600, 0, 0, 2.0, 6.0, 1, G.ptr(out), G.stream()), "pack_rays")
    got = out.cpu().numpy()
    np.testing.assert_allclose(got[:, 0:3], fx["rays_o"].reshape(-1, 3), atol=1e-6)
    np.testing.assert_allclose(got[:, 3:6], fx["rays_d"].reshape(-1, 3), atol=1e-6)
    assert np.all(got[:, 6] == 2.0) and np.all(got[:, 7] == 6.0)
    d = fx["rays_d"].reshape(-1, 3)
    np.testing.assert_allclose(got[:, 8:11], d / np.linalg.norm(d, axis=-1, keepdims=True), atol=1e-6)
    # 2. fern-shaped rays with NDC == reference ndc_rays
    c2wf = G.synth.fern_camera()[3]
    cam = _camera(38, 50, fx["ndc_K"], c2wf)
    out = torch.empty((38 * 50, 11), device=G.DEV)
    G._lib.check(lib.nerf_b200_pack_rays(None, None, None, C.byref(cam), 38 * 50, 0, 1, 0.0, 1.0, 1, G.ptr(out), G.stream()), "pack_rays")
    got = out.cpu().numpy()
    np.testing.assert_allclose(got[:, 0:3], fx["ndc_o"].reshape(-1, 3), atol=2e-6)
    np.testing.assert_allclose(got[:, 3:6], fx["ndc_d"].reshape(-1, 3), atol=2e-6)
    # 3. explicit rays in == oracle pack_rays (both NDC settings), 8-wide rows without viewdirs
    sb = G.synth.ray_batch("fern", 333, seed=2)
    for ndc in (False, True):
        for uv in (True, False):
            ref = G.O.pack_rays(sb["H"], sb["W"], sb["K"], sb["rays"][0], sb["rays"][1], ndc, 0.25, 1.5, uv)
            o, dd = G.dev(sb["rays"][0]), G.dev(sb["rays"][1])
            cam = _camera(sb["H"], sb["W"], sb["K"])
            out = torch.empty((333, 11 if uv else 8), device=G.DEV)
            G._lib.check(lib.nerf_b200_pack_rays(G.ptr(o), G.ptr(dd), None, C.byref(cam), 333, 0, int(ndc), 0.25, 1.5, int(uv), G.ptr(out), G.stream()), "pack_rays")
            np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=2e-6, atol=2e-6)


def test_render_c2w_full_image_path(G):
    """render(c2w=...) (render_path's call, run_nerf.py:154): in-kernel ray generation == explicit rays."""
    H, W, K, c2w = G.synth.lego_camera(24)
    nets = [G.make_net(G.synth.nerf_state(0)), G.make_net(G.synth.nerf_state(1))]
    kw = dict(ndc=False, near=2., far=6., use_viewdirs=True, network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(),
              N_samples=64, N_importance=128, perturb=0., white_bkgd=True, raw_noise_std=0.)
    o, d = G.synth.camera_rays(H, W, K, c2w)
    with torch.no_grad():
        a = G.nb.render(H, W, K, chunk=300, c2w=torch.from_numpy(c2w).to(G.DEV), **kw)
        b = G.nb.render(H, W, K, chunk=32768, rays=(G.dev(o), G.dev(d)), **kw)
    assert a[0].shape == (H, W, 3) and a[1].shape == (H, W)
    torch.testing.assert_close(a[0], b[0], rtol=2e-4, atol=2e-5)
