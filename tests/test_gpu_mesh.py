"""Mesh extraction on the GPU: density_grid, marching_cubes, extract_mesh.

(a) density_grid = run_network(meshgrid points, zero viewdirs)[..., 3] bit for bit, in tc_fp16, tc_split and fp32, at every
    tensor-core shape of test_gpu_shapes.SHAPES (with and without view directions), at shapes only the exact path serves (fp32),
    on grids with odd sizes, nz = 2, nz > 256 (a column over several tiles), more columns than one wave of CTAs, and (fp32)
    more points than one slab of the exact path;
(b) density_grid against the reference's own run_network (tests/golden/density_grid.npz): fp32 and tc_split within the exact
    path's raw gate, tc_fp16 within the tensor-core raw gate of test_gpu_shapes;
(c) the GPU marching cubes against the numpy restatement (tests/mc_emul.py): identical faces, bit-identical vertices, on a
    sphere, a torus and a trained net's density at several levels, with cells at sigma == iso exactly and NaN corners;
(d) run-to-run bits of sigma, verts and faces;
(e) extract_mesh end to end on the trained fine net: each vertex interpolates its edge's densities to iso;
(f) refusals: a net the precision refuses is rejected before any launch, with run_network's message; emit refuses outputs
    smaller than the counts and a workspace counted for another grid."""

import numpy as np
import pytest
import torch

import mc_emul as M
from conftest import load_golden, rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


@pytest.fixture(autouse=True)
def _restore_precision():
    import nerf_pytorch_b200 as nb
    yield
    nb.set_precision("tc_fp16")


def _axes(shape, seed, lo=-1.5, hi=1.5):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(np.sort(rng.uniform(lo, hi, n)).astype(np.float32)).cuda() for n in shape]


def _query(L, Lv):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.api import _QueryFn
    i_embed = 0 if L > 0 else -1
    e, _ = nb.get_embedder(L, i_embed)
    ed, _ = nb.get_embedder(Lv, i_embed) if Lv else (None, 0)
    return _QueryFn(e, ed, 65536, L, Lv, i_embed)


def _via_run_network(net, q, xs, ys, zs, views):
    import nerf_pytorch_b200 as nb
    pts = torch.stack(torch.meshgrid(xs, ys, zs, indexing="ij"), -1)
    nx, ny, nz = pts.shape[:3]
    vd = torch.zeros((nx * ny, 3), device=pts.device) if views else None
    raw = nb.run_network(pts.reshape(nx * ny, nz, 3), vd, net, q.embed_fn, q.embeddirs_fn)
    return raw[..., 3].reshape(nx, ny, nz)


def _bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


GRIDS = [(7, 5, 13), (33, 31, 2), (3, 2, 300), (181, 97, 3)]       # odd; nz = 2; nz > 256; 17557 columns


def _shapes():
    import test_gpu_shapes as S
    return S.SHAPES


@pytest.mark.parametrize("prec", ["tc_fp16", "tc_split", "fp32"])
@pytest.mark.parametrize("shape", _shapes(), ids=[s[0] for s in _shapes()])
def test_density_grid_is_run_network_bit_for_bit(G, prec, shape):
    import nerf_pytorch_b200 as nb
    import test_gpu_shapes as S
    sid, D, skips, L, Lv, out_ch, seed = shape
    sh = S._shape(G, sid, D, skips, L, Lv, out_ch, seed=seed)
    q = _query(sh.L, sh.Lv)
    nb.set_precision(prec)
    for g, shp in enumerate(GRIDS):
        xs, ys, zs = _axes(shp, g)
        got = nb.density_grid(sh.net, q, xs, ys, zs)
        ref = _via_run_network(sh.net, q, xs, ys, zs, sh.views)
        assert got.shape == shp and torch.isfinite(got).all(), (sid, shp)
        assert np.array_equal(_bits(got), _bits(ref)), (sid, prec, shp, float((got - ref).abs().max()))


EXACT_ONLY = [("w100", 100, 8, [4], 10, 4), ("d10", 256, 10, [4], 10, 4), ("L14", 256, 8, [4], 14, 4), ("w100_nv", 100, 6, [2], 10, None)]


@pytest.mark.parametrize("case", EXACT_ONLY, ids=[c[0] for c in EXACT_ONLY])
def test_density_grid_exact_only_shapes(G, case):
    import nerf_pytorch_b200 as nb
    import test_gpu_shapes as S
    sid, W, D, skips, L, Lv = case
    sh = S._shape(G, sid, D, skips, L, Lv, 5, seed=1, W=W)
    q = _query(sh.L, sh.Lv)
    nb.set_precision("fp32")
    grids = GRIDS + ([(104, 103, 100)] if sid == "w100" else [])        # > 2^20 points: several slabs
    for g, shp in enumerate(grids):
        xs, ys, zs = _axes(shp, 10 + g)
        got, ref = nb.density_grid(sh.net, q, xs, ys, zs), _via_run_network(sh.net, q, xs, ys, zs, sh.views)
        assert np.array_equal(_bits(got), _bits(ref)), (sid, shp)
    if W != 256:
        launches = nb.launch_count()
        nb.set_precision("tc_fp16")
        with pytest.raises(RuntimeError, match=r"set_precision\('fp32'\)"):
            nb.density_grid(sh.net, q, xs, ys, zs)
        assert nb.launch_count() == launches


def _trained(G):
    from oracle import outgrads
    w = load_golden("trained_weights")
    st = [{k[2:]: v for k, v in w.items() if k.startswith(t + ".")} for t in ("c", "f")]
    nv = G.make_net(outgrads.noviews_from_trained(st[1], 1), use_viewdirs=False, output_ch=5)
    return {"c": G.make_net(st[0]), "f": G.make_net(st[1]), "nv": nv}


@pytest.mark.parametrize("prec", ["tc_fp16", "tc_split", "fp32"])
def test_density_grid_against_the_reference(G, prec):
    import nerf_pytorch_b200 as nb
    fx = load_golden("density_grid")
    nets = _trained(G)
    nb.set_precision(prec)
    xs, ys, zs = (G.dev(fx[k]) for k in ("xs", "ys", "zs"))
    for tag, net in nets.items():
        q = _query(10, 4 if tag != "nv" else 0)
        got = nb.density_grid(net, q, xs, ys, zs).cpu().numpy()
        assert np.isfinite(got).all()
        err = rel_l2(got, fx[tag + "_sigma64"])
        cond = rel_l2(fx[tag + "_sigma"], fx[tag + "_sigma64"])
        gate = 2e-3 if prec == "tc_fp16" else 2e-5 + 2 * cond
        print(prec, tag, "rel-L2 vs reference float64 %.3g (reference float32 %.3g)" % (err, cond))
        assert err < gate, (prec, tag, err, cond)


def _mc(sigma, xs, ys, zs, iso):
    import nerf_pytorch_b200 as nb
    v, f = nb.marching_cubes(sigma, xs, ys, zs, iso)
    ve, fe = M.marching_cubes(sigma.cpu().numpy(), xs.cpu().numpy(), ys.cpu().numpy(), zs.cpu().numpy(), iso)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    assert f.dtype == np.int64 and np.array_equal(f, fe), (iso, f.shape, fe.shape)
    assert v.shape == ve.shape and np.array_equal(np.isnan(v), np.isnan(ve))
    ok = ~np.isnan(ve)
    assert np.array_equal(v[ok].view(np.int32), ve[ok].view(np.int32)), iso
    return v, f


def test_marching_cubes_matches_the_restatement(G):
    import nerf_pytorch_b200 as nb
    a = torch.linspace(-1, 1, 48, device="cuda")
    X, Y, Z = torch.meshgrid(a, a, a, indexing="ij")
    sphere = 0.7 - torch.sqrt(X * X + Y * Y + Z * Z)
    v, f = _mc(sphere, a, a, a, 0.0)
    assert set(M.edge_counts(f).tolist()) == {2} and M.euler(v, f) == 2 and M.signed_volume(v, f) > 0
    torus = 0.25 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 0.6) ** 2 + Z * Z)
    v, f = _mc(torus, a, a, a, 0.0)
    assert set(M.edge_counts(f).tolist()) == {2} and M.euler(v, f) == 0
    # a trained net's density on a non-uniform grid, at several levels; then with cells at sigma == iso and NaN corners
    xs, ys, zs = _axes((40, 37, 45), 3, -1.3, 1.3)
    sigma = nb.density_grid(_trained(G)["f"], _query(10, 4), xs, ys, zs)
    for iso in (0.0, 5.0, 10.0):
        v, f = _mc(sigma, xs, ys, zs, iso)
        print("iso", iso, "verts", len(v), "faces", len(f))
        assert len(f) > 100, iso
    # NaN beside inside points (their edges cross: t is NaN there), and inside points set to the level exactly (outside)
    s2 = sigma.clone()
    inside = torch.nonzero((s2[:, :, :-1] > 0.0).reshape(-1)).reshape(-1)
    assert len(inside) > 300
    pick = inside[torch.randperm(len(inside), generator=torch.Generator().manual_seed(0))[:300].cuda()]
    i, jk = pick // ((s2.shape[1]) * (s2.shape[2] - 1)), pick % ((s2.shape[1]) * (s2.shape[2] - 1))
    j, k = jk // (s2.shape[2] - 1), jk % (s2.shape[2] - 1)
    s2[i[:150], j[:150], k[:150] + 1] = float("nan")
    s2[i[150:], j[150:], k[150:]] = 0.0
    v, f = _mc(s2, xs, ys, zs, 0.0)
    assert np.isnan(v).any() and len(f) > 0


def test_run_to_run_bits(G):
    import nerf_pytorch_b200 as nb
    net, q = _trained(G)["f"], _query(10, 4)
    xs, ys, zs = _axes((64, 64, 64), 5, -1.3, 1.3)
    for prec in ("tc_fp16", "tc_split", "fp32"):
        nb.set_precision(prec)
        s1, s2 = nb.density_grid(net, q, xs, ys, zs), nb.density_grid(net, q, xs, ys, zs)
        assert np.array_equal(_bits(s1), _bits(s2)), prec
        (v1, f1), (v2, f2) = nb.marching_cubes(s1, xs, ys, zs, 0.0), nb.marching_cubes(s1, xs, ys, zs, 0.0)
        assert len(f1) > 100 and np.array_equal(_bits(v1), _bits(v2)) and torch.equal(f1, f2), prec


def test_extract_mesh_end_to_end(G, tmp_path):
    import nerf_pytorch_b200 as nb
    net, q = _trained(G)["f"], _query(10, 4)
    xs, ys, zs = _axes((72, 70, 68), 6, -1.3, 1.3)
    iso = 5.0
    v, f = nb.extract_mesh(net, q, xs, ys, zs, iso)
    sigma = nb.density_grid(net, q, xs, ys, zs).cpu().numpy().astype(np.float64)
    assert len(f) > 100 and f.min() >= 0 and f.max() < len(v)
    # vertex ids follow the crossing edges in C order, then axis: recompute each vertex's edge and interpolate along it
    inside = sigma > iso
    act = np.zeros(sigma.shape + (3,), bool)
    act[:-1, :, :, 0] = inside[:-1] != inside[1:]
    act[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    act[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    pi, pj, pk, ax = np.nonzero(act)
    assert len(ax) == len(v)
    v = v.cpu().numpy().astype(np.float64)
    axes = [a.cpu().numpy().astype(np.float64) for a in (xs, ys, zs)]
    lo = np.stack([pi, pj, pk], 1)
    hi = lo + np.eye(3, dtype=np.int64)[ax]
    sa, sb = sigma[tuple(lo.T)], sigma[tuple(hi.T)]
    ca = np.array([axes[a][lo[n, a]] for n, a in enumerate(ax)])
    cb = np.array([axes[a][hi[n, a]] for n, a in enumerate(ax)])
    c = v[np.arange(len(v)), ax]
    s = sa + (c - ca) / (cb - ca) * (sb - sa)
    eps = np.finfo(np.float32).eps
    tol = 4 * eps * (np.abs(sb - sa) * (np.abs(c) + np.abs(ca) + np.abs(cb)) / np.abs(cb - ca) + abs(iso) + np.abs(sa))
    assert np.all(np.abs(s - iso) <= tol), float(np.max(np.abs(s - iso) / tol))
    nb.save_ply(str(tmp_path / "mesh.ply"), v, f)


def test_refusals_before_any_launch(G):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib
    import test_gpu_shapes as S
    sh = S._shape(G, "w128", 8, [4], 10, 4, 5, seed=0, W=128)
    q = _query(10, 4)
    xs, ys, zs = _axes((5, 6, 7), 0)
    pts = torch.stack(torch.meshgrid(xs, ys, zs, indexing="ij"), -1).reshape(30, 7, 3)
    for prec in ("tc_fp16", "tc_split"):
        nb.set_precision(prec)
        with pytest.raises(RuntimeError) as rn:
            nb.run_network(pts, torch.zeros(30, 3, device="cuda"), sh.net, q.embed_fn, q.embeddirs_fn)
        launches = nb.launch_count()
        with pytest.raises(RuntimeError) as dg:
            nb.density_grid(sh.net, q, xs, ys, zs)
        assert nb.launch_count() == launches
        assert str(dg.value) == str(rn.value) and "set_precision('fp32')" in str(dg.value)
    # emit: outputs below the counts, and a workspace counted for another grid or level
    lib = _lib.load()
    a = torch.linspace(-1, 1, 16, device="cuda")
    X, Y, Z = torch.meshgrid(a, a, a, indexing="ij")
    sigma = (0.6 - torch.sqrt(X * X + Y * Y + Z * Z)).contiguous()
    wsb = lib.nerf_b200_marching_cubes_workspace_bytes(16, 16, 16)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    counts = torch.empty(2, dtype=torch.int64, device="cuda")
    p = G.ptr
    _lib.check(lib.nerf_b200_marching_cubes_count(p(sigma), 16, 16, 16, 0.0, p(counts), p(ws), wsb, G.stream()), "count")
    V, F = counts.tolist()
    verts = torch.empty((V, 3), device="cuda")
    faces = torch.empty((F, 3), dtype=torch.int32, device="cuda")
    launches = nb.launch_count()
    for args, msg in (((V - 1, F, 0.0), "outputs too small"), ((V, F - 1, 0.0), "outputs too small"), ((V, F, 0.5), "another grid or iso")):
        rc = lib.nerf_b200_marching_cubes_emit(p(sigma), p(a), p(a), p(a), 16, 16, 16, args[2], p(verts), args[0], p(faces), args[1],
                                               p(ws), wsb, G.stream())
        assert rc != 0 and msg in lib.nerf_b200_last_error().decode(), msg
    assert nb.launch_count() == launches
    _lib.check(lib.nerf_b200_marching_cubes_emit(p(sigma), p(a), p(a), p(a), 16, 16, 16, 0.0, p(verts), V, p(faces), F, p(ws), wsb,
                                                 G.stream()), "emit")
    torch.cuda.synchronize()
    assert np.array_equal(faces.long().cpu().numpy(), M.marching_cubes(sigma.cpu().numpy(), a.cpu().numpy(), a.cpu().numpy(), a.cpu().numpy(), 0.0)[1])
