"""Mesh extraction without a GPU: the marching-cubes rules on the numpy restatement (tests/mc_emul.py, which reads the library's
triangle table from mesh.cuh), the argument validation of the new C entry points, the PLY writer and the density fixture.

  * sphere f = R - |p| on a 48^3 grid: closed (every edge in two faces), Euler characteristic 2, vertices within 0.1 h of the
    sphere, positive signed volume (normals outward) within 2 % of 4/3 pi R^3;
  * torus: closed, Euler characteristic 0;
  * every one of the 256 single-cell configurations: the table's triangle count, vertices only on edges whose ends differ;
  * random fields (outside on the border): closed and consistently wound, every directed edge once -- the table is consistent
    between neighbouring cells, including its ambiguous faces;
  * every new entry point refuses bad arguments before it launches or dereferences anything (fake pointers);
  * save_ply reads back to the same arrays.
"""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import mc_emul as M
from conftest import GOLDEN, load_golden


def _grid(n, lo=-1.0, hi=1.0):
    a = np.linspace(lo, hi, n, dtype=np.float32)
    return a, np.meshgrid(a, a, a, indexing="ij")


def _closed(faces):
    return set(M.edge_counts(faces).tolist()) == {2}


def test_sphere():
    a, (X, Y, Z) = _grid(48)
    R = 0.7
    f = (R - np.sqrt(X * X + Y * Y + Z * Z)).astype(np.float32)
    v, fc = M.marching_cubes(f, a, a, a, 0.0)
    h = float(a[1] - a[0])
    assert len(fc) > 1000 and _closed(fc)
    assert M.euler(v, fc) == 2
    assert np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - R).max() < 0.1 * h
    vol = M.signed_volume(v, fc)
    assert vol > 0 and abs(vol - 4 / 3 * np.pi * R ** 3) < 0.02 * 4 / 3 * np.pi * R ** 3, vol


def test_torus():
    a, (X, Y, Z) = _grid(48)
    f = (0.25 - np.sqrt((np.sqrt(X * X + Y * Y) - 0.6) ** 2 + Z * Z)).astype(np.float32)
    v, fc = M.marching_cubes(f, a, a, a, 0.0)
    assert _closed(fc) and M.euler(v, fc) == 0
    assert M.signed_volume(v, fc) > 0


def test_every_single_cell_configuration():
    a = np.array([0.0, 1.0], np.float32)
    counts = set()
    for case in range(256):
        # corner v outside (bit set) -> sigma -1, inside -> +1, at the grid point of its offset
        s = np.empty((2, 2, 2), np.float32)
        for v, (dx, dy, dz) in enumerate(M.CORNERS):
            s[dx, dy, dz] = -1.0 if (case >> v) & 1 else 1.0
        v, fc = M.marching_cubes(s, a, a, a, 0.0)
        assert len(fc) == M.NTRI[case], case
        counts.add(len(fc))
        # every vertex is the midpoint of an edge whose ends differ: two coordinates on the grid, one at 0.5
        assert np.all(np.sum(v == 0.5, axis=1) == 1) and np.all(np.isin(v, (0.0, 0.5, 1.0))), case
        for p in v:
            lo, hi = np.floor(p).astype(int), np.ceil(p).astype(int)
            assert (s[tuple(lo)] > 0) != (s[tuple(hi)] > 0), (case, p)
        if len(fc):
            assert len(np.unique(fc)) == len(v)          # every vertex is used
    assert counts == {0, 1, 2, 3, 4, 5}


@pytest.mark.parametrize("seed", range(4))
def test_random_fields_are_closed_and_consistently_wound(seed):
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((14, 13, 12)).astype(np.float32)
    g[[0, -1]] = -1; g[:, [0, -1]] = -1; g[:, :, [0, -1]] = -1
    v, fc = M.marching_cubes(g, np.arange(14, dtype=np.float32), np.arange(13, dtype=np.float32), np.arange(12, dtype=np.float32), 0.0)
    assert len(fc) > 200 and _closed(fc)
    directed = np.concatenate([fc[:, [0, 1]], fc[:, [1, 2]], fc[:, [2, 0]]])
    assert len(np.unique(directed, axis=0)) == len(directed)


def test_nan_and_level_values_are_outside():
    a = np.array([0.0, 1.0], np.float32)
    s = np.full((2, 2, 2), np.nan, np.float32)
    s[0, 0, 0] = 1.0
    v, fc = M.marching_cubes(s, a, a, a, 0.0)
    assert len(fc) == 1 and np.isnan(v).any()              # t is NaN on an edge to a NaN corner
    s[:] = 0.5
    assert len(M.marching_cubes(s, a, a, a, 0.5)[1]) == 0   # sigma == iso everywhere: all outside


def test_save_ply_round_trip(tmp_path):
    import nerf_pytorch_b200 as nb
    a, (X, Y, Z) = _grid(12)
    v, fc = M.marching_cubes((0.6 - np.sqrt(X * X + Y * Y + Z * Z)).astype(np.float32), a, a, a, 0.0)
    path = os.path.join(tmp_path, "m.ply")
    nb.save_ply(path, v, fc)
    raw = open(path, "rb").read()
    head, body = raw.split(b"end_header\n", 1)
    assert f"element vertex {len(v)}".encode() in head and f"element face {len(fc)}".encode() in head
    v2 = np.frombuffer(body[:12 * len(v)], "<f4").reshape(-1, 3)
    rec = np.frombuffer(body[12 * len(v):], dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    assert np.array_equal(v2, v) and np.all(rec["n"] == 3) and np.array_equal(rec["idx"], fc)


def test_density_fixture_belongs_to_the_trained_weights():
    fx = load_golden("density_grid")
    digest = hashlib.sha256(open(os.path.join(GOLDEN, "trained_weights.npz"), "rb").read()).digest()
    assert bytes(fx["weights_sha256"]) == digest
    assert fx["f_sigma"].shape == (len(fx["xs"]), len(fx["ys"]), len(fx["zs"]))
    assert all(np.all(np.diff(fx[k]) > 0) for k in ("xs", "ys", "zs"))
    # the density crosses 0 inside the grid
    assert all(fx[k + "_sigma"].min() < 0 < fx[k + "_sigma"].max() for k in ("c", "f", "nv"))


# ---- refusals ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from nerf_pytorch_b200 import _lib
    return _lib


def test_new_entry_points_refuse_during_argument_validation(lib):
    """Every refusal happens before a launch or a dereference: the pointers are fake."""
    L = lib.load()
    fake = C.c_void_p(256)
    tc = lib.NerfNetParams(D=8, W=256, skip=4, input_ch=63, input_ch_views=27, use_viewdirs=1, output_ch=4)
    w128 = lib.NerfNetParams(D=8, W=128, skip=4, input_ch=63, input_ch_views=27, use_viewdirs=1, output_ch=4)
    w50 = lib.NerfNetParams(D=8, W=50, skip=4, input_ch=63, input_ch_views=27, use_viewdirs=1, output_ch=4)
    launches = L.nerf_b200_launch_count()

    def dg(net, prec, xs=fake, nx=4, mr=10, packed=fake, ws=fake, wsb=1 << 30):
        return L.nerf_b200_density_grid(xs, nx, fake, 5, fake, 6, C.byref(net), packed, mr, prec, fake, ws, wsb, None)

    def mc_count(nx=4, sigma=fake, ws=fake, wsb=1 << 30):
        return L.nerf_b200_marching_cubes_count(sigma, nx, 5, 6, 0.0, fake, ws, wsb, None)

    def mc_emit(nx=4, verts=fake, mv=10, ws=fake, wsb=1 << 30):
        return L.nerf_b200_marching_cubes_emit(fake, fake, fake, fake, nx, 5, 6, 0.0, verts, mv, fake, 10, ws, wsb, None)

    cases = {
        "density NULL axis": (lambda: dg(tc, lib.PREC_TC_FP16, xs=None), "NULL pointer"),
        "density empty grid": (lambda: dg(tc, lib.PREC_TC_FP16, nx=0), "empty grid"),
        "density unknown precision": (lambda: dg(tc, 7), "unknown precision"),
        "density tc width": (lambda: dg(w128, lib.PREC_TC_FP16), "set_precision('fp32')"),
        "density split width": (lambda: dg(w128, lib.PREC_TC_SPLIT), "set_precision('fp32')"),
        "density exact width": (lambda: dg(w50, lib.PREC_FP32), "netwidth <= 256 and a multiple of 4"),
        "density multires": (lambda: dg(tc, lib.PREC_TC_FP16, mr=9), "multires 9 does not match input_ch 63"),
        "density packed": (lambda: dg(tc, lib.PREC_TC_FP16, packed=None), "call nerf_b200_pack_weights"),
        "density split packed": (lambda: dg(tc, lib.PREC_TC_SPLIT, packed=None), "call nerf_b200_pack_weights_split"),
        "density exact workspace": (lambda: dg(w128, lib.PREC_FP32, wsb=16), "workspace too small"),
        "count nx": (lambda: mc_count(nx=1), "nx, ny, nz >= 2"),
        "count NULL": (lambda: mc_count(sigma=None), "NULL pointer"),
        "count workspace": (lambda: mc_count(wsb=64), "workspace too small"),
        "count huge": (lambda: L.nerf_b200_marching_cubes_count(fake, 2048, 2048, 2048, 0.0, fake, fake, 1 << 62, None), "too large"),
        "emit nx": (lambda: mc_emit(nx=1), "nx, ny, nz >= 2"),
        "emit NULL verts": (lambda: mc_emit(verts=None), "NULL output"),
        "emit negative": (lambda: mc_emit(mv=-1), "NULL output"),
        "emit workspace": (lambda: mc_emit(wsb=64), "workspace too small"),
    }
    for name, (call, msg) in cases.items():
        rc = call()
        err = L.nerf_b200_last_error().decode()
        assert rc != 0 and msg in err, (name, err)
    # the refusal of the tensor-core precisions is run_network's, word for word
    L.nerf_b200_run_network(fake, fake, 8, 16, C.byref(w128), fake, 10, 4, lib.PREC_TC_FP16, fake, fake, 1 << 30, None)
    rn_msg = L.nerf_b200_last_error().decode()
    dg(w128, lib.PREC_TC_FP16)
    assert L.nerf_b200_last_error().decode() == rn_msg
    assert L.nerf_b200_launch_count() == launches
    # workspace sizes: 0 where refused
    assert L.nerf_b200_density_grid_workspace_bytes(4, 5, 6, C.byref(w128), lib.PREC_TC_FP16) == 0
    assert L.nerf_b200_density_grid_workspace_bytes(4, 5, 6, C.byref(w128), lib.PREC_FP32) > 4 * 5 * 6 * 28
    assert L.nerf_b200_density_grid_workspace_bytes(4, 5, 6, C.byref(tc), lib.PREC_TC_SPLIT) > 0
    assert L.nerf_b200_marching_cubes_workspace_bytes(1, 5, 6) == 0
    assert L.nerf_b200_marching_cubes_workspace_bytes(4, 5, 6) >= 4 * 5 * 6 * 8
