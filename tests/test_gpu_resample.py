"""Hierarchical sampling on the GPU equals the reference bit for bit, through the C ABI: nerf_b200_sample_pdf,
nerf_b200_fine_z, and both coarse-z producers (coarse_z_kernel and, inside nerf_b200_render_rays_fwd at tensor-core
precision, ray_setup_kernel).  References: tests/golden/resample.npz and trained_lego_1024.npz (the unmodified reference
on CPU torch) and oracle/resample.py, which tests/test_resample_cpu.py pins to both."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import resample as R
from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


def bits_equal(got, ref):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    assert got.shape == ref.shape
    bad = got.view(np.uint32) != ref.view(np.uint32)
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0]}: {got[bad][0]} vs {ref[bad][0]}"


def sample_pdf(G, bins, w, u, n):
    """nerf_b200_sample_pdf; u is a shared [n] row (row stride 0) or [N, n]."""
    N, B = bins.shape
    d_b, d_w, d_u = G.dev(bins), G.dev(w), G.dev(u)
    out = torch.full((N, n), float("nan"), device=G.DEV)
    G._lib.check(G._lib.load().nerf_b200_sample_pdf(G.ptr(d_b), G.ptr(d_w), G.ptr(d_u), 0 if u.ndim == 1 else n, N, B, n,
                                                    G.ptr(out), G.stream()), "sample_pdf")
    return out.cpu().numpy()


def fine_z(G, z, w, u, n_imp, want_samples=True, want_std=True):
    """nerf_b200_fine_z -> (z_fine, z_samples | None, z_std | None)"""
    N, S = z.shape
    d_z, d_w, d_u = G.dev(z), G.dev(w), G.dev(u)
    zf = torch.full((N, S + n_imp), float("nan"), device=G.DEV)
    zs = torch.full((N, n_imp), float("nan"), device=G.DEV) if want_samples else None
    sd = torch.full((N,), float("nan"), device=G.DEV) if want_std else None
    G._lib.check(G._lib.load().nerf_b200_fine_z(G.ptr(d_z), G.ptr(d_w), G.ptr(d_u), 0 if u.ndim == 1 else n_imp, N, S, n_imp,
                                                G.ptr(zf), G.ptr(zs), G.ptr(sd), G.stream()), "fine_z")
    return zf.cpu().numpy(), (zs.cpu().numpy() if zs is not None else None), (sd.cpu().numpy() if sd is not None else None)


def axis_rays(near, far, stride=8):
    """rays from the origin along +z with per-ray near / far (and +z view directions)"""
    r = np.zeros((len(near), stride), np.float32)
    r[:, 5], r[:, 6], r[:, 7] = 1.0, near, far
    if stride == 11:
        r[:, 10] = 1.0
    return r


def coarse_z_kernel(G, rays, S, lindisp, t_rand):
    N = rays.shape[0]
    d_r, d_t = G.dev(rays), torch.linspace(0., 1., S, device=G.DEV)
    d_tr = G.dev(t_rand) if t_rand is not None else None
    z = torch.full((N, S), float("nan"), device=G.DEV)
    G._lib.check(G._lib.load().nerf_b200_coarse_z(G.ptr(d_r), rays.shape[1], G.ptr(d_t), G.ptr(d_tr), N, S, lindisp, G.ptr(z),
                                                  G.stream()), "coarse_z")
    return z.cpu().numpy()


_NET = {}


def ray_setup_z(G, rays11, S, lindisp, t_rand):
    """z_coarse of nerf_b200_render_rays_fwd at tensor-core precision (ray_setup_kernel), coarse pass only"""
    lib = G._lib.load()
    if "c" not in _NET:
        _NET["c"] = G.make_net(synth.nerf_state(0))
    net = _NET["c"]
    N = rays11.shape[0]
    cfg = G._lib.NerfRenderCfg()
    cfg.N_samples, cfg.N_importance, cfg.multires, cfg.multires_views = S, 0, 10, 4
    cfg.lindisp, cfg.perturb, cfg.white_bkgd, cfg.ray_stride = lindisp, int(t_rand is not None), 1, 11
    cfg.precision = G._lib.PREC_TC_FP16
    zc, rgb, acc = (torch.zeros(s, device=G.DEV) for s in ((N, S), (N, 3), (N,)))
    out = G._lib.NerfPassOut(G.ptr(rgb), C.c_void_p(0), G.ptr(acc), C.c_void_p(0), C.c_void_p(0), C.c_void_p(0))
    p = net.net_params()
    ws_bytes = lib.nerf_b200_march_workspace_bytes(N, S)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=G.DEV)
    d_r, d_t = G.dev(rays11), torch.linspace(0., 1., S, device=G.DEV)
    d_tr = G.dev(t_rand) if t_rand is not None else None
    G._lib.check(lib.nerf_b200_render_rays_fwd(G.ptr(d_r), N, C.byref(cfg), C.byref(p), G.ptr(net.packed()), None, None,
                                               G.ptr(d_t), None, G.ptr(d_tr), None, None, None, G.ptr(zc), C.byref(out), None, None,
                                               None, G.ptr(ws), ws_bytes, G.stream()), "render_rays_fwd")
    return zc.cpu().numpy()


def weights_for(rng, N, n):
    """[N, n] coarse-weight rows: random, cubed, opaque (a peak, then exact zeros), all zero, in turn"""
    w = rng.random((N, n), dtype=np.float32)
    w[1::4] **= 3
    k = n // 3
    w[2::4, k + 1:] = 0.0
    w[2::4, k] = 0.9
    w[3::4] = 0.0
    return w


# ---- linspace ----------------------------------------------------------------------------------------------------

def test_cuda_linspace_equals_cpu():
    """t_vals and det u are built with torch.linspace on the device; the reference builds them on CPU."""
    for n in (1, 2, 3, 8, 31, 32, 33, 64, 65, 128, 192, 596, 960, 1000, 1024, 2048, 3500, 4096):
        bits_equal(torch.linspace(0., 1., n, device="cuda").cpu().numpy(), torch.linspace(0., 1., n).numpy())


# ---- the reference's own outputs ---------------------------------------------------------------------------------

def _ids(prefix):
    fx = load_golden("resample")
    return sorted(int(k[1:-5]) for k in fx if k.startswith(prefix) and k.endswith("_meta"))


@pytest.mark.parametrize("i", _ids("p"))
def test_sample_pdf_golden(G, i):
    fx = load_golden("resample")
    B, n, kind = (int(v) for v in fx[f"p{i}_meta"])
    bins, w, u, ref = fx[f"p{i}_bins"], fx[f"p{i}_w"], fx[f"p{i}_u"], fx[f"p{i}_out"]
    bits_equal(sample_pdf(G, bins, w, u, n), ref)
    if kind in (0, 1):            # the Python entry point draws the det row itself (torch.linspace, or np.linspace under pytest)
        bits_equal(G.nb.sample_pdf(G.dev(bins), G.dev(w), n, det=True, pytest=kind == 1).cpu().numpy(), ref)


@pytest.mark.parametrize("i", _ids("f"))
def test_fine_z_and_coarse_z_golden(G, i):
    fx = load_golden("resample")
    p = f"f{i}_"
    S, Ni, lindisp, perturb = (int(v) for v in fx[p + "meta"])
    t_rand = fx.get(p + "t_rand")
    bits_equal(coarse_z_kernel(G, axis_rays(fx[p + "near"], fx[p + "far"]), S, lindisp, t_rand), fx[p + "z_coarse"])
    bits_equal(ray_setup_z(G, axis_rays(fx[p + "near"], fx[p + "far"], 11), S, lindisp, t_rand), fx[p + "z_coarse"])
    u = fx[p + "u"] if perturb else R.torch_linspace(Ni)
    zf, zs, sd = fine_z(G, fx[p + "z_coarse"], fx[p + "w_coarse"], u, Ni)
    bits_equal(zf, fx[p + "z_fine"])
    bits_equal(sd, fx[p + "z_std"])
    bits_equal(zs, R.sample_pdf(0.5 * (fx[p + "z_coarse"][:, 1:] + fx[p + "z_coarse"][:, :-1]), fx[p + "w_coarse"][:, 1:-1], Ni, u=u))


def test_trained_lego_1024(G):
    """The reference's coarse weights of 1024 trained-net rays: fine_z reproduces its z_fine and z_std, and both z producers
    its z_coarse."""
    fx = load_golden("trained_lego_1024")
    N = fx["z_coarse"].shape[0]
    near, far = np.full(N, 2.0, np.float32), np.full(N, 6.0, np.float32)
    bits_equal(coarse_z_kernel(G, axis_rays(near, far), 64, 0, None), fx["z_coarse"])
    bits_equal(ray_setup_z(G, axis_rays(near, far, 11), 64, 0, None), fx["z_coarse"])
    zf, _, sd = fine_z(G, fx["z_coarse"], fx["w_coarse"], R.torch_linspace(128), 128)
    bits_equal(zf, fx["z_fine"])
    bits_equal(sd, fx["z_std"])


# ---- the accepted range against the restatement ------------------------------------------------------------------

@pytest.mark.parametrize("S,lindisp,perturb", [(1, 0, 0), (1, 0, 1), (2, 1, 1), (3, 0, 1), (64, 1, 0), (1024, 0, 1), (1024, 1, 1)])
def test_coarse_z_both_producers(G, S, lindisp, perturb):
    rng = np.random.default_rng(S * 4 + lindisp * 2 + perturb)
    N = 37
    near = (0.5 + 2 * rng.random(N, dtype=np.float32)).astype(np.float32)
    far = (near + 0.5 + 6 * rng.random(N, dtype=np.float32)).astype(np.float32)
    t_rand = None
    if perturb:
        t_rand = rng.random((N, S), dtype=np.float32)
        t_rand[::3] = 0.0
        t_rand[1::3] = 1.0
        t_rand[2, 0] = 1.0
    ref = R.coarse_z(near[:, None], far[:, None], S, bool(lindisp), t_rand)
    bits_equal(coarse_z_kernel(G, axis_rays(near, far), S, lindisp, t_rand), ref)
    bits_equal(ray_setup_z(G, axis_rays(near, far, 11), S, lindisp, t_rand), ref)


# (S, n_imp, N, u): S + n_imp at a power of two (128), one past it (129) and 4096, including S past 3478, where four rays'
# rows no longer fit one block's shared memory; u "det" (a shared linspace row) and "sorted" take the binary-search
# merge, "rand" the counting merge
FINE_MATRIX = [(3, 1, 5, "det"), (97, 31, 4, "rand"), (96, 32, 3, "sorted"), (96, 33, 1025, "det"), (64, 128, 1025, "rand"),
               (64, 128, 5, "sorted"), (136, 960, 5, "det"), (3136, 960, 3, "rand"), (3500, 596, 5, "sorted"),
               (4095, 1, 4, "det"), (3968, 128, 5, "rand"), (1000, 1, 1025, "rand")]


@pytest.mark.parametrize("S,n_imp,N,ukind", FINE_MATRIX)
def test_fine_z_matrix(G, S, n_imp, N, ukind):
    rng = np.random.default_rng(S * 7 + n_imp)
    z = np.sort(2 + 4 * rng.random((N, S), dtype=np.float32), -1).astype(np.float32)
    z[:, 1:3] = z[:, 1:2]                                   # a tie among the coarse z
    w = weights_for(rng, N, S)
    if ukind == "det":
        u = R.torch_linspace(n_imp)
    else:
        u = rng.random((N, n_imp), dtype=np.float32)
        if n_imp >= 2:
            u[:, :2] = [0.0, 1.0]
        if ukind == "sorted":
            u = np.sort(u, -1)
    ref_f, ref_s, ref_sd = R.fine_z(z, w, n_imp, u=u)
    zf, zs, sd = fine_z(G, z, w, u, n_imp)
    bits_equal(zf, ref_f)
    bits_equal(zs, ref_s)
    bits_equal(sd, ref_sd)
    zf2, _, _ = fine_z(G, z, w, u, n_imp, want_samples=False, want_std=False)
    bits_equal(zf2, ref_f)


@pytest.mark.parametrize("B,n,N", [(2, 33, 5), (7, 128, 4), (65, 1, 3), (513, 128, 1025), (600, 64, 5), (1100, 31, 5), (2048, 128, 5)])
def test_sample_pdf_matrix(G, B, n, N):
    rng = np.random.default_rng(B * 3 + n)
    bins = np.sort(2 + 4 * rng.random((N, B), dtype=np.float32), -1).astype(np.float32)
    w = weights_for(rng, N, B - 1)
    u = rng.random((N, n), dtype=np.float32)
    u[:, 0] = 1.0
    bits_equal(sample_pdf(G, bins, w, u, n), R.sample_pdf(bins, w, n, u=u))
    row = R.torch_linspace(n)
    bits_equal(sample_pdf(G, bins, w, row, n), R.sample_pdf(bins, w, n, u=row))


def test_fine_z_refuses_what_the_reference_cannot_do(G):
    """S = 2 leaves sample_pdf no weights (the reference's torch.gather fails on its empty cdf); S + n_imp > 4096 is
    beyond the kernel's per-ray row."""
    z = np.tile(np.float32([2.0, 6.0]), (3, 1))
    with pytest.raises(RuntimeError):
        fine_z(G, z, np.ones_like(z), R.torch_linspace(8), 8)
    z = np.sort(np.random.default_rng(0).random((2, 4000), dtype=np.float32), -1)
    with pytest.raises(RuntimeError):
        fine_z(G, z, np.ones_like(z), R.torch_linspace(97), 97)
