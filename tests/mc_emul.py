"""A numpy restatement of the library's marching cubes (nerf-pytorch_b200/csrc/mesh.cuh), written from the rules, not the kernels:

  * a grid point is inside when sigma > iso (NaN: outside); cube case bit v is set when corner v is not inside;
  * one vertex per grid edge whose ends differ, ids in grid-point C order then axis x, y, z;
  * the vertex on the edge a -> b (a the lower index) along an axis: t = (iso - s_a) / (s_b - s_a), c = c_a + t (c_b - c_a), each
    step rounded to float32 (numpy float32 arithmetic is IEEE round-to-nearest and never fuses);
  * faces in cell C order then table order, each as the table lists its edges (normals toward decreasing density).

The triangle table is read from mesh.cuh, so the tests below check the table the library is built with."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MESH_CUH = os.path.join(ROOT, "nerf-pytorch_b200", "csrc", "mesh.cuh")

# corner v -> (dx, dy, dz); cube edge -> (corner a, corner b)
CORNERS = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]])
EDGES = np.array([[0, 1], [1, 2], [3, 2], [0, 3], [4, 5], [5, 6], [7, 6], [4, 7], [0, 4], [1, 5], [2, 6], [3, 7]])


def tri_table():
    """[256, 16] int array of mesh.cuh's mc_tri_table"""
    src = open(MESH_CUH).read()
    body = src[src.index("mc_tri_table[256][16] = {"):]
    body = body[body.index("{") + 1:body.index("};")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{([^{}]*)\}", body)]
    t = np.array(rows, dtype=np.int64)
    assert t.shape == (256, 16), t.shape
    return t


TRI = tri_table()
NTRI = np.array([int(np.sum(r >= 0)) // 3 for r in TRI])


def marching_cubes(sigma, xs, ys, zs, iso):
    """-> (verts [V, 3] float32, faces [F, 3] int64)"""
    sigma = np.asarray(sigma, np.float32)
    xs, ys, zs = (np.asarray(a, np.float32) for a in (xs, ys, zs))
    iso = np.float32(iso)
    nx, ny, nz = sigma.shape
    with np.errstate(invalid="ignore"):
        inside = sigma > iso
    # active edges per point and axis, and the vertex ids
    act = np.zeros((nx, ny, nz, 3), bool)
    act[:-1, :, :, 0] = inside[:-1] != inside[1:]
    act[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    act[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = act.reshape(-1)
    vid = np.full(flat.shape, -1, np.int64)
    vid[flat] = np.arange(int(flat.sum()))
    vid = vid.reshape(nx, ny, nz, 3)
    # positions
    pi, pj, pk, ax = np.nonzero(act)
    d = np.stack([(ax == 0), (ax == 1), (ax == 2)], 1).astype(np.int64)
    sa = sigma[pi, pj, pk]
    sb = sigma[pi + d[:, 0], pj + d[:, 1], pk + d[:, 2]]
    with np.errstate(invalid="ignore", divide="ignore"):
        t = (iso - sa) / (sb - sa)
    axes = (xs, ys, zs)
    idx = (pi, pj, pk)
    verts = np.empty((len(ax), 3), np.float32)
    for a in range(3):
        ca = axes[a][idx[a]]
        cb = axes[a][np.minimum(idx[a] + d[:, a], len(axes[a]) - 1)]
        with np.errstate(invalid="ignore"):
            lerp = ca + t * (cb - ca)
        verts[:, a] = np.where(ax == a, lerp, ca)
    # cases
    out = ~inside
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for v, (dx, dy, dz) in enumerate(CORNERS):
        case |= out[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz].astype(np.int64) << v
    faces = []
    ci, cj, ck = np.nonzero(NTRI[case] > 0)
    cases = case[ci, cj, ck]
    for t_ in range(5):
        has = NTRI[cases] > t_
        e = TRI[cases[has]][:, 3 * t_:3 * t_ + 3]
        ids = []
        for c in range(3):
            a_ = CORNERS[EDGES[e[:, c], 0]]
            b_ = CORNERS[EDGES[e[:, c], 1]]
            axis = np.argmax(b_ - a_, axis=1)
            ids.append(vid[ci[has] + a_[:, 0], cj[has] + a_[:, 1], ck[has] + a_[:, 2], axis])
        faces.append((ci[has], cj[has], ck[has], t_, np.stack(ids, 1)))
    # cell C order, then table order
    if not faces:
        return verts, np.zeros((0, 3), np.int64)
    cell = np.concatenate([(f[0] * (ny - 1) + f[1]) * (nz - 1) + f[2] for f in faces])
    tt = np.concatenate([np.full(len(f[0]), f[3]) for f in faces])
    tri = np.concatenate([f[4] for f in faces])
    order = np.lexsort((tt, cell))
    return verts, tri[order]


def edge_counts(faces):
    """{undirected edge: number of faces that have it}"""
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    e = np.sort(e, axis=1)
    _, c = np.unique(e, axis=0, return_counts=True)
    return c


def euler(verts, faces):
    e = np.unique(np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1), axis=0)
    return len(np.unique(faces)) - len(e) + len(faces)


def signed_volume(verts, faces):
    v = verts.astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(np.sum(np.einsum("ij,ij->i", a, np.cross(b, c))) / 6.0)
