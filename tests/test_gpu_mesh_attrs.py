"""Vertex attributes on the GPU: density_gradient, vertex_attributes, save_ply with normals and colours.

(a) the gradient against a float64 autograd of the same network (tests/test_mesh_attrs_cpu.ref_sigma_grad) at every shape of
    test_gpu_shapes.SHAPES and at the exact-only shapes of its section (e), gated at 1e-4 plus twice the float32 autograd's own
    distance from float64 (the exact backward's gradient gate); (b) at the same shapes sigma is run_network(pts)[..., 3] in fp32
    bit for bit;
(c) the same bits in tc_fp16, tc_split and fp32 and from run to run, at P = 1, an odd P and P over several slabs, on workspaces
    of 0xFF bytes and of zeros;
(d) against the reference (tests/golden/vertex_attrs.npz): the gradient within (a)'s gate of its float64 autograd; the colours
    within test_gpu_mesh.py (b)'s precision classes; vertex_attributes' colours bit for bit sigmoid(run_network(...)) in every
    precision;
(e) extract_mesh + vertex_attributes: normals of unit length or zero, colours in [0, 1]; on a smooth net at least 90 % of vertices
    agree in sign with their area-weighted face normal (marching_cubes' winding), on the trained fine net the share is recorded;
    the mesh is written with both attributes;
(f) refusals: a net the exact path refuses (its message, no launch), a workspace that is too small, CPU tensors.

Measured values go to parity_mesh_attrs.json in $NERF_B200_PARITY_DIR (default: a nerf_b200_parity directory under the system's
temporary directory)."""
import ctypes as C
import json
import os
import re
import tempfile

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2
from test_mesh_attrs_cpu import ref_sigma_grad, relu_margin

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


def _record(name, value):
    out_dir = os.environ.get("NERF_B200_PARITY_DIR") or os.path.join(tempfile.gettempdir(), "nerf_b200_parity")
    path = os.path.join(out_dir, "parity_mesh_attrs.json")
    os.makedirs(out_dir, exist_ok=True)
    data = json.load(open(path)) if os.path.isfile(path) else {}
    data[name] = value
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def _query(L, Lv):
    from test_gpu_mesh import _query as q
    return q(L, Lv)


def _trained(G):
    from test_gpu_mesh import _trained as t
    return t(G)


def _bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


def _points(P, seed, lo=-1.5, hi=1.5):
    return torch.from_numpy(np.random.default_rng(seed).uniform(lo, hi, (P, 3)).astype(np.float32)).cuda()


def _shape_cases():
    import test_gpu_shapes as S
    tc = [(sid, 256, D, skips, L, Lv, out_ch, seed) for sid, D, skips, L, Lv, out_ch, seed in S.SHAPES]
    ex = [(sid, W, D, skips, L, Lv, out_ch, seed) for sid, W, D, skips, L, Lv, out_ch, _, _, seed in S.EXACT_SHAPES]
    return tc + ex


def _check_against_float64(state, pts, L, Lv, views, grad, stats, tag):
    """rel-L2 against float64 autograd at 1e-4 plus twice float32 autograd's distance, on the points where no pre-activation is
    within 1e-6 of its scale of 0: at a ReLU kink the gradient jumps, and the forward's rounding picks the side"""
    p = pts.cpu().numpy()
    keep = relu_margin(state, p, L, Lv, views) > 1e-6
    stats[tag + "_at_kink"] = int((~keep).sum())
    assert keep.mean() > 0.95, (tag, stats)
    _, g64 = ref_sigma_grad(state, p[keep], L, Lv, views)
    _, g32 = ref_sigma_grad(state, p[keep], L, Lv, views, torch.float32)
    g = grad.cpu().numpy()
    assert np.isfinite(g).all(), tag
    e, cond = rel_l2(g[keep], g64), rel_l2(g32, g64)
    stats[tag + "_grad_rel"], stats[tag + "_cond"] = e, cond
    assert e < 1e-4 + 2 * cond, (tag, e, cond)


@pytest.mark.parametrize("case", _shape_cases(), ids=[c[0] for c in _shape_cases()])
def test_gradient_against_float64(G, case):
    import nerf_pytorch_b200 as nb
    import test_gpu_shapes as S
    sid, W, D, skips, L, Lv, out_ch, seed = case
    sh = S._shape(G, sid, D, skips, L, Lv, out_ch, seed=seed, W=W)
    q = _query(sh.L, sh.Lv)
    pts = _points(777, seed)
    sigma, grad = nb.density_gradient(sh.net, q, pts)
    assert sigma.shape == (777,) and grad.shape == (777, 3)
    stats = {}
    _check_against_float64(sh.state, pts, sh.L, sh.Lv, sh.views, grad, stats, sid)
    # (b) sigma is run_network's in fp32, bit for bit, whatever the view directions
    nb.set_precision("fp32")
    vd = torch.nn.functional.normalize(_points(777, seed + 1), dim=-1) if sh.views else None
    raw = nb.run_network(pts[:, None], vd, sh.net, q.embed_fn, q.embeddirs_fn)
    assert np.array_equal(_bits(sigma), _bits(raw[:, 0, 3])), sid
    _record(f"shape_{sid}", stats)


def _c_call(G, net, pts, L, fill):
    """nerf_b200_density_gradient on a workspace filled with byte `fill` -> (sigma, grad)"""
    from nerf_pytorch_b200 import _lib
    lib = _lib.load()
    n = net.net_params()
    P = pts.shape[0]
    wsb = lib.nerf_b200_density_gradient_workspace_bytes(P, C.byref(n))
    ws = torch.full((wsb,), fill, dtype=torch.uint8, device="cuda")
    sigma, grad = torch.empty(P, device="cuda"), torch.empty((P, 3), device="cuda")
    _lib.check(lib.nerf_b200_density_gradient(G.ptr(pts), P, C.byref(n), L, G.ptr(sigma), G.ptr(grad), G.ptr(ws), wsb, G.stream()),
               "density_gradient")
    torch.cuda.synchronize()
    return sigma, grad


@pytest.mark.parametrize("P", [1, 4097, 40000], ids=["P1", "P_odd", "P_three_slabs"])
def test_same_bits_in_every_precision_and_run(G, P):
    import nerf_pytorch_b200 as nb
    net, q = _trained(G)["f"], _query(10, 4)
    pts = _points(P, P, -1.3, 1.3)
    ref = None
    for prec in ("tc_fp16", "tc_split", "fp32"):
        nb.set_precision(prec)
        for out in (nb.density_gradient(net, q, pts), _c_call(G, net, pts, 10, 0xFF), _c_call(G, net, pts, 10, 0)):
            got = (_bits(out[0]), _bits(out[1]))
            if ref is None:
                ref = got
                assert np.isfinite(out[1].cpu().numpy()).all()
            assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), (prec, P)


@pytest.mark.parametrize("prec", ["tc_fp16", "tc_split", "fp32"])
def test_against_the_reference(G, prec):
    import nerf_pytorch_b200 as nb
    fx = load_golden("vertex_attrs")
    nets = _trained(G)
    nb.set_precision(prec)
    stats = {}
    for tag, net in nets.items():
        views = tag != "nv"
        q = _query(10, 4 if views else 0)
        pts = G.dev(fx[tag + "_pts"])
        sigma, grad = nb.density_gradient(net, q, pts)
        g = grad.cpu().numpy()
        assert np.isfinite(g).all()
        e, cond = rel_l2(g, fx[tag + "_grad64"]), rel_l2(fx[tag + "_grad"], fx[tag + "_grad64"])
        stats[tag + "_grad_rel"], stats[tag + "_grad_cond"] = e, cond
        assert e < 1e-4 + 2 * cond, (tag, e, cond)
        normals, colors = nb.vertex_attributes(net, q, pts)
        # the colours are sigmoid(run_network) in this precision, bit for bit
        n = grad.norm(dim=-1, keepdim=True)
        look = torch.where(n > 0, grad / n, torch.zeros_like(grad))
        raw = nb.run_network(pts[:, None], look if views else None, net, q.embed_fn, q.embeddirs_fn)
        assert np.array_equal(_bits(colors), _bits(torch.sigmoid(raw[:, 0, :3]))), tag
        assert np.array_equal(_bits(normals), _bits(-look)), tag
        c = colors.cpu().numpy()
        e, cond = rel_l2(c, fx[tag + "_colors64"]), rel_l2(fx[tag + "_colors"], fx[tag + "_colors64"])
        stats[tag + "_colors_rel"], stats[tag + "_colors_cond"] = e, cond
        gate = 2e-3 if prec == "tc_fp16" else 2e-5 + 2 * cond
        print(prec, tag, "gradient rel-L2 %.3g (reference float32 %.3g), colours %.3g (%.3g)"
              % (stats[tag + "_grad_rel"], stats[tag + "_grad_cond"], e, cond))
        assert e < gate, (prec, tag, e, cond)
    _record(f"reference_{prec}", stats)


def _share_along_face_normals(v, f, normals):
    """the share of vertices whose normal has a positive dot product with the area-weighted sum of their faces' normals"""
    vv, ff = v.cpu().numpy().astype(np.float64), f.cpu().numpy()
    fn = np.cross(vv[ff[:, 1]] - vv[ff[:, 0]], vv[ff[:, 2]] - vv[ff[:, 0]])
    acc = np.zeros_like(vv)
    for k in range(3):
        np.add.at(acc, ff[:, k], fn)
    return float(np.mean(np.sum(acc * normals.cpu().numpy().astype(np.float64), 1) > 0))


def _check_normals_and_colors(normals, colors):
    length = np.linalg.norm(normals.cpu().numpy().astype(np.float64), axis=1)
    assert np.all((np.abs(length - 1) < 1e-5) | (length == 0))
    c = colors.cpu().numpy()
    assert np.isfinite(c).all() and c.min() >= 0 and c.max() <= 1
    return int(np.sum(length == 0))


def test_mesh_end_to_end(G, tmp_path):
    """The sign convention against marching_cubes' winding (faces toward decreasing density) on a smooth field: a net without
    encoding (multires 0, i_embed = -1), whose density is piecewise linear at the scale of the grid.  Then the trained fine net at
    iso 10, whose top octave (period 0.0123) is far below a 96^3 grid's spacing (0.027): its normals follow the network's fine
    structure, not the facets, and the share is recorded and only required to beat a flipped sign."""
    import nerf_pytorch_b200 as nb
    import test_gpu_shapes as S
    xs = torch.linspace(-1.3, 1.3, 96, device="cuda")
    sh = S._shape(G, "smooth", 4, [], 0, 0, 5, seed=3, W=64)
    q0 = _query(0, 0)
    nb.set_precision("fp32")
    iso = float(nb.density_grid(sh.net, q0, xs, xs, xs).median())
    v, f = nb.extract_mesh(sh.net, q0, xs, xs, xs, iso)
    normals, colors = nb.vertex_attributes(sh.net, q0, v)
    smooth = {"V": len(v), "F": len(f), "zero_normals": _check_normals_and_colors(normals, colors),
              "positive_share": _share_along_face_normals(v, f, normals)}
    nb.set_precision("tc_fp16")
    net, q = _trained(G)["f"], _query(10, 4)
    v, f = nb.extract_mesh(net, q, xs, xs, xs, 10.0)
    normals, colors = nb.vertex_attributes(net, q, v)
    trained = {"V": len(v), "F": len(f), "zero_normals": _check_normals_and_colors(normals, colors),
               "positive_share": _share_along_face_normals(v, f, normals)}
    _record("end_to_end", {"smooth": smooth, "trained_fine_iso10": trained})
    print("smooth net", smooth, "trained fine net", trained)
    assert smooth["F"] > 1000 and smooth["positive_share"] >= 0.9, smooth
    assert trained["F"] > 1000 and trained["positive_share"] > 0.5, trained
    path = str(tmp_path / "mesh.ply")
    nb.save_ply(path, v, f, normals, colors)
    head = open(path, "rb").read().split(b"end_header\n", 1)[0].decode()
    assert "property float nx" in head and "property uchar red" in head and f"element vertex {len(v)}" in head


def test_refusals(G):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib
    lib = _lib.load()
    q = _query(10, 4)
    pts = _points(100, 0)
    bad = nb.NeRF(D=2, W=50, input_ch=63, input_ch_views=27, output_ch=5, skips=[], use_viewdirs=True).cuda()
    nb.set_precision("fp32")
    with pytest.raises(RuntimeError) as rn:
        nb.run_network(pts[:, None], torch.zeros(100, 3, device="cuda"), bad, q.embed_fn, q.embeddirs_fn)
    for prec in ("tc_fp16", "fp32"):
        nb.set_precision(prec)
        launches = nb.launch_count()
        for fn in (nb.density_gradient, nb.vertex_attributes):
            with pytest.raises(RuntimeError, match=re.escape("a multiple of 4")) as dg:
                fn(bad, q, pts)
            assert str(dg.value).split("): ", 1)[1] == str(rn.value).split("): ", 1)[1]
        assert nb.launch_count() == launches
    # a workspace one byte short
    net = _trained(G)["f"]
    n = net.net_params()
    wsb = lib.nerf_b200_density_gradient_workspace_bytes(100, C.byref(n))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    out = torch.empty((100, 4), device="cuda")
    launches = nb.launch_count()
    rc = lib.nerf_b200_density_gradient(G.ptr(pts), 100, C.byref(n), 10, G.ptr(out), G.ptr(out), G.ptr(ws), wsb - 1, G.stream())
    assert rc != 0 and "workspace too small" in lib.nerf_b200_last_error().decode()
    assert nb.launch_count() == launches
    # CPU tensors
    for fn in (nb.density_gradient, nb.vertex_attributes):
        with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
            fn(net, q, pts.cpu())
    # no points, no launch
    s, g = nb.density_gradient(net, q, pts[:0])
    assert s.shape == (0,) and g.shape == (0, 3) and nb.launch_count() == launches
