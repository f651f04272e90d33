"""Vertex attributes without a GPU: the references the GPU tests compare the density gradient against, the argument validation of
nerf_b200_density_gradient, and save_ply's normals and colours.

  * a float64 autograd of oracle/torch_ref (embed + mlp) on the fixture's points reproduces the reference's own float64 autograd
    through its run_network (tests/golden/vertex_attrs.npz, `<n>_grad64`): this pins the restatement tests/test_gpu_mesh_attrs.py
    compares against;
  * the encoding's Jacobian as csrc/bwd_simt.cuh's enc_jacobian_kernel forms it, restated in numpy, matches float64 central
    differences of the encoding (identity only when L = 0);
  * the library exports the new entry points, and every refusal comes before a launch or a dereference (fake pointers);
  * save_ply with normals and colours reads back exactly; without them its bytes are the plain writer's.
"""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden, rel_l2


def ref_sigma_grad(state, pts, L, Lv, views, dtype=torch.float64):
    """sigma and dsigma/dx of oracle/torch_ref's network at pts [P, 3] by autograd in `dtype` (zero view directions)"""
    from oracle import torch_ref as T
    sd = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in state.items()}
    x = torch.from_numpy(np.asarray(pts)).to(dtype).requires_grad_(True)
    enc = T.embed(x, L)
    ic = enc.shape[1]
    icv = 0
    if views:
        encv = T.embed(torch.zeros_like(x), Lv)
        icv = encv.shape[1]
        enc = torch.cat([enc, encv], -1)
    D = sum(1 for k in sd if k.startswith("pts_linears.") and k.endswith(".weight"))
    skip = next((i for i in range(D - 1) if sd[f"pts_linears.{i + 1}.weight"].shape[1] != sd["pts_linears.1.weight"].shape[0]), -1)
    sigma = T.mlp(sd, enc, ic=ic, icv=icv, skip=skip, D=D)[:, 3]
    (g,) = torch.autograd.grad(sigma.sum(), x)
    return sigma.detach().numpy(), g.numpy()


def relu_margin(state, pts, L, Lv, views):
    """per point, the least |a| / (|b| + sum_k |w_k h_k|) over every pts-layer pre-activation a = b + sum_k w_k h_k, in float64:
    where it is within float32 rounding of 0 the ReLU's side, and so the gradient, is decided by the rounding of the forward"""
    from oracle import torch_ref as T
    sd = {k: np.asarray(v, np.float64) for k, v in state.items()}
    x = torch.from_numpy(np.asarray(pts, np.float64))
    enc = T.embed(x, L).numpy()
    D = sum(1 for k in sd if k.startswith("pts_linears.") and k.endswith(".weight"))
    h, out = enc, np.full(len(enc), np.inf)
    for i in range(D):
        w, b = sd[f"pts_linears.{i}.weight"], sd[f"pts_linears.{i}.bias"]
        if w.shape[1] != h.shape[1]:                       # the layer after the skip reads cat([input_pts, h])
            h = np.concatenate([enc, h], 1)
        a = h @ w.T + b
        out = np.minimum(out, (np.abs(a) / (np.abs(b) + np.abs(h) @ np.abs(w).T)).min(1))
        h = np.maximum(a, 0)
    return out


def _trained_states():
    from oracle import outgrads
    c, f = outgrads.trained_states(os.path.join(GOLDEN, "trained_weights.npz"))
    return {"c": (c, True), "f": (f, True), "nv": (outgrads.noviews_from_trained(f, 1), False)}


def test_fixture_belongs_to_the_trained_weights():
    fx = load_golden("vertex_attrs")
    digest = hashlib.sha256(open(os.path.join(GOLDEN, "trained_weights.npz"), "rb").read()).digest()
    assert bytes(fx["weights_sha256"]) == digest
    nu = int(fx["n_uniform"])
    for n in ("c", "f", "nv"):
        P = len(fx[n + "_pts"])
        assert P > nu + 500 and fx[n + "_grad64"].shape == (P, 3) and fx[n + "_colors"].shape == (P, 3)
        # the near-surface points straddle the level 0 of the net's density
        s = fx[n + "_sigma"][nu:]
        assert np.abs(s).max() < 0.5 * np.abs(fx[n + "_sigma"][:nu]).max()


@pytest.mark.parametrize("net", ["c", "f", "nv"])
def test_restatement_reproduces_the_reference_autograd(net):
    fx = load_golden("vertex_attrs")
    state, views = _trained_states()[net]
    sigma, g = ref_sigma_grad(state, fx[net + "_pts"], 10, 4, views)
    assert rel_l2(g, fx[net + "_grad64"]) < 1e-12, rel_l2(g, fx[net + "_grad64"])
    assert rel_l2(sigma, fx[net + "_sigma"]) < 1e-6
    s32, g32 = ref_sigma_grad(state, fx[net + "_pts"], 10, 4, views, torch.float32)
    assert rel_l2(g32, fx[net + "_grad64"]) < 1e-5


def _enc_jacobian(d_enc, x, L):
    """enc_jacobian_kernel in numpy (float64): d_enc [P, 3 + 6 L], x [P, 3] -> [P, 3]"""
    g = d_enc[:, 0:3].copy()
    for k in range(L):
        a = x * 2.0 ** k
        g += 2.0 ** k * (np.cos(a) * d_enc[:, 3 + 6 * k:6 + 6 * k] - np.sin(a) * d_enc[:, 6 + 6 * k:9 + 6 * k])
    return g


@pytest.mark.parametrize("L", [0, 1, 4, 10, 16])
def test_encoding_jacobian_matches_central_differences(L):
    from oracle import torch_ref as T
    rng = np.random.default_rng(L)
    P = 64
    x = rng.uniform(-1.3, 1.3, (P, 3))
    d_enc = rng.standard_normal((P, 3 + 6 * L))
    got = _enc_jacobian(d_enc, x, L)
    h = 1e-4 / 2.0 ** max(L - 1, 0)                     # a step well inside the top octave's period
    fd = np.zeros((P, 3))
    for j in range(3):
        e = np.zeros(3)
        e[j] = h
        fp = (T.embed(torch.from_numpy(x + e), L).numpy() * d_enc).sum(-1)
        fm = (T.embed(torch.from_numpy(x - e), L).numpy() * d_enc).sum(-1)
        fd[:, j] = (fp - fm) / (2 * h)
    assert rel_l2(got, fd) < 1e-6, rel_l2(got, fd)
    if L == 0:
        assert np.array_equal(got, d_enc)


# ---- the C entry points ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from nerf_pytorch_b200 import _lib
    return _lib


def test_entry_points_are_exported(lib):
    so = C.CDLL(lib.LIB_PATH)
    for name in ("nerf_b200_density_gradient", "nerf_b200_density_gradient_workspace_bytes"):
        assert hasattr(so, name) and name in lib.SIGNATURES, name
    header = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "nerf_b200.h")).read()
    assert "nerf_b200_density_gradient(" in header and "nerf_b200_density_gradient_workspace_bytes(" in header


def test_density_gradient_refuses_during_argument_validation(lib):
    """Every refusal happens before a launch or a dereference: the pointers are fake."""
    L = lib.load()
    fake = C.c_void_p(256)
    net = lib.NerfNetParams(D=8, W=256, skip=4, input_ch=63, input_ch_views=27, use_viewdirs=1, output_ch=4)
    w50 = lib.NerfNetParams(D=8, W=50, skip=4, input_ch=63, input_ch_views=27, use_viewdirs=1, output_ch=4)
    skip_last = lib.NerfNetParams(D=4, W=64, skip=3, input_ch=63, input_ch_views=27, use_viewdirs=1, output_ch=4)
    launches = L.nerf_b200_launch_count()
    need = L.nerf_b200_density_gradient_workspace_bytes(1000, C.byref(net))
    assert need > 1000 * (2 * 63 + 8 * 256 + 2 * 256 + 4) * 4

    def dg(n=net, P=1000, pts=fake, sigma=fake, grad=fake, mr=10, ws=fake, wsb=need):
        return L.nerf_b200_density_gradient(pts, P, C.byref(n), mr, sigma, grad, ws, wsb, None)

    cases = {
        "NULL pts": (lambda: dg(pts=None), "NULL pointer"),
        "NULL sigma": (lambda: dg(sigma=None), "NULL pointer"),
        "NULL grad": (lambda: dg(grad=None), "NULL pointer"),
        "NULL workspace": (lambda: dg(ws=None), "NULL pointer"),
        "negative P": (lambda: dg(P=-1), "P must be >= 0"),
        "width": (lambda: dg(n=w50), "netwidth <= 256 and a multiple of 4"),
        "skip after the last layer": (lambda: dg(n=skip_last), "skip layer must be < netdepth - 1"),
        "multires": (lambda: dg(mr=9), "multires 9 does not match input_ch 63"),
        "workspace": (lambda: dg(wsb=need - 1), "workspace too small"),
        "alignment": (lambda: dg(ws=C.c_void_p(264)), "16-byte boundary"),
    }
    for name, (call, msg) in cases.items():
        rc = call()
        err = L.nerf_b200_last_error().decode()
        assert rc != 0 and msg in err, (name, err)
    # the width refusal is the exact path's, word for word (nerf_b200_run_network in FP32)
    L.nerf_b200_run_network(fake, fake, 8, 16, C.byref(w50), None, 10, 4, lib.PREC_FP32, fake, None, 0, None)
    rn_msg = L.nerf_b200_last_error().decode()
    dg(n=w50)
    assert L.nerf_b200_last_error().decode() == rn_msg
    assert dg(P=0) == 0                                    # nothing to do
    assert L.nerf_b200_launch_count() == launches
    # workspace: 0 where refused; bounded by one slab for any P
    assert L.nerf_b200_density_gradient_workspace_bytes(10, C.byref(w50)) == 0
    assert L.nerf_b200_density_gradient_workspace_bytes(-1, C.byref(net)) == 0
    slab = L.nerf_b200_density_gradient_workspace_bytes(1 << 14, C.byref(net))
    assert L.nerf_b200_density_gradient_workspace_bytes(1 << 40, C.byref(net)) == slab
    assert slab == 512 + (1 << 14) * (2 * 63 + 8 * 256 + 2 * 256 + 4) * 4


def test_python_surface_refuses_cpu_tensors(lib):
    import nerf_pytorch_b200 as nb
    net = nb.NeRF(D=2, W=64, input_ch=63, input_ch_views=27, output_ch=5, skips=[], use_viewdirs=True)
    e, _ = nb.get_embedder(10, 0)
    ed, _ = nb.get_embedder(4, 0)
    from nerf_pytorch_b200.api import _QueryFn
    q = _QueryFn(e, ed, 65536, 10, 4, 0)
    for fn in (nb.density_gradient, nb.vertex_attributes):
        with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
            fn(net, q, torch.zeros(5, 3))


# ---- save_ply ---------------------------------------------------------------------------------------------------------------

def _plain_ply(path, v, f):
    """the PLY writer without vertex attributes, as it was before normals and colours: the bytes save_ply must keep"""
    v = np.ascontiguousarray(v, dtype="<f4").reshape(-1, 3)
    rec = np.empty(len(f), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    rec["n"] = 3
    rec["idx"] = np.asarray(f).reshape(-1, 3)
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {len(v)}\nproperty float x\nproperty float y\n"
              f"property float z\nelement face {len(rec)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii") + v.tobytes() + rec.tobytes())


def _mesh():
    import mc_emul as M
    a = np.linspace(-1, 1, 12, dtype=np.float32)
    X, Y, Z = np.meshgrid(a, a, a, indexing="ij")
    return M.marching_cubes((0.6 - np.sqrt(X * X + Y * Y + Z * Z)).astype(np.float32), a, a, a, 0.0)


def test_save_ply_without_attributes_is_unchanged(tmp_path):
    import nerf_pytorch_b200 as nb
    v, f = _mesh()
    nb.save_ply(str(tmp_path / "a.ply"), v, f)
    _plain_ply(str(tmp_path / "b.ply"), v, f)
    assert open(tmp_path / "a.ply", "rb").read() == open(tmp_path / "b.ply", "rb").read()
    nb.save_ply(str(tmp_path / "c.ply"), torch.from_numpy(v), torch.from_numpy(f))
    assert open(tmp_path / "c.ply", "rb").read() == open(tmp_path / "b.ply", "rb").read()


@pytest.mark.parametrize("which", ["normals", "colors", "both"])
def test_save_ply_with_attributes_round_trip(tmp_path, which):
    import nerf_pytorch_b200 as nb
    v, f = _mesh()
    rng = np.random.default_rng(1)
    nrm = rng.standard_normal(v.shape).astype(np.float32)
    col = rng.uniform(-0.2, 1.2, v.shape).astype(np.float32)          # out of [0, 1] on purpose: to8b clips
    kw = {"normals": nrm if which != "colors" else None, "colors": torch.from_numpy(col) if which != "normals" else None}
    path = str(tmp_path / "m.ply")
    nb.save_ply(path, v, f, **kw)
    head, body = open(path, "rb").read().split(b"end_header\n", 1)
    props = [ln.split()[-1] for ln in head.decode().splitlines() if ln.startswith("property") and "list" not in ln]
    fields = [("p", "<f4", (3,))]
    want = ["x", "y", "z"]
    if kw["normals"] is not None:
        fields.append(("n", "<f4", (3,)))
        want += ["nx", "ny", "nz"]
    if kw["colors"] is not None:
        fields.append(("c", "u1", (3,)))
        want += ["red", "green", "blue"]
    assert props == want
    assert (b"property uchar red" in head) == (kw["colors"] is not None)
    vd = np.dtype(fields)
    vr = np.frombuffer(body[:vd.itemsize * len(v)], dtype=vd)
    rec = np.frombuffer(body[vd.itemsize * len(v):], dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    assert np.array_equal(vr["p"], v) and np.all(rec["n"] == 3) and np.array_equal(rec["idx"], f)
    if kw["normals"] is not None:
        assert np.array_equal(vr["n"], nrm)
    if kw["colors"] is not None:
        assert np.array_equal(vr["c"], nb.to8b(col)) and vr["c"].dtype == np.uint8
