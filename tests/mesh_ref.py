"""Serial numpy float32 restatement of the surface extraction (DESIGN.md §6j), the checker of i3d_mesh.cuh.

Written from the reference's semantics (MarchingCubes::extractMesh / extractSurfaceAt / getVertex / interpolate / merge,
MeshUtil::removeDegenerateFaces / removeLooseComponents / removeUnusedVertices) with the generated case tables.  It shares no code
with the kernels: welding is a dict keyed on float tuples (as merge's std::map), components come from scipy.sparse.csgraph.
"""
import os
import sys

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "intrinsic3d_b200", "csrc"))
import gen_mc_tables  # noqa: E402

EDGE_MASK, TRIS = gen_mc_tables.tables()
CORNERS = np.array(gen_mc_tables.CORNERS, np.int64)
EDGES = gen_mc_tables.EDGES
F32 = np.float32


def _keys(xyz):
    x = xyz.astype(np.int64) + (1 << 20)
    return (x[:, 0] << 42) | (x[:, 1] << 21) | x[:, 2]


def _interp(s0, s1, v0, v1):
    """interpolate(tsdf0, tsdf1, val0, val1, 0.0f) row-wise in float32: v0, v1 [m, 3]."""
    zero, eps = F32(0), F32(1e-5)
    with np.errstate(divide="ignore", invalid="ignore"):
        mu = (zero - s0) / (s1 - s0)
    mu = np.where(F32(1) < mu, F32(1), mu)
    mu = np.where(mu < zero, zero, mu)
    lerp = v0 + mu[:, None] * (v1 - v0)
    end0 = (np.abs(zero - s0) < eps) | ((np.abs(zero - s1) >= eps) & (np.abs(s0 - s1) < eps))
    end1 = ~(np.abs(zero - s0) < eps) & (np.abs(zero - s1) < eps)
    return np.where(end0[:, None], v0, np.where(end1[:, None], v1, lerp)).astype(F32)


def marching_cubes(xyz, sdf, weight, rgb, voxel_size):
    """Triangle soup in (voxel index, triangle slot) order: corner positions float32 [F, 3, 3], colours uint8 [F, 3, 3], number of used
    cubes."""
    xyz = np.asarray(xyz, np.int32)
    sdf = np.asarray(sdf, np.float64)
    weight = np.asarray(weight, np.float32)
    rgb = np.asarray(rgb, np.uint8)
    n = len(xyz)
    keys = _keys(xyz)
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    idx = np.empty((n, 8), np.int64)
    for c in range(8):
        q = _keys(xyz.astype(np.int64) + CORNERS[c])
        pos = np.clip(np.searchsorted(sk, q), 0, max(n - 1, 0))
        found = sk[pos] == q if n else np.zeros(0, bool)
        idx[:, c] = np.where(found, order[pos], -1)
    valid = (idx >= 0).all(1)
    valid[valid] = (weight[idx[valid]] != 0).all(1)
    case = np.zeros(n, np.int64)
    for c in range(8):
        case[valid] |= (sdf[idx[valid, c]] < 0.0).astype(np.int64) << c
    vs = F32(voxel_size)
    inv255 = F32(1) / F32(255)
    pos_out, col_out = [], []
    for v in np.nonzero(valid & (case != 0) & (case != 255))[0]:
        tris = TRIS[case[v]]
        if not tris:
            continue
        ends = np.array([EDGES[e] for t in tris for e in t])             # [3T, 2] corner numbers
        ia, ib = idx[v, ends[:, 0]], idx[v, ends[:, 1]]
        s0, s1 = sdf[ia].astype(F32), sdf[ib].astype(F32)
        p0 = (xyz[v].astype(np.int64) + CORNERS[ends[:, 0]]).astype(F32) * vs
        p1 = (xyz[v].astype(np.int64) + CORNERS[ends[:, 1]]).astype(F32) * vs
        c0 = rgb[ia].astype(F32) * inv255
        c1 = rgb[ib].astype(F32) * inv255
        p = _interp(s0, s1, p0, p1)
        col = (_interp(s0, s1, c0, c1) * F32(255)).astype(np.uint8)
        pos_out.append(p.reshape(-1, 3, 3))
        col_out.append(col.reshape(-1, 3, 3))
    if not pos_out:
        return np.zeros((0, 3, 3), F32), np.zeros((0, 3, 3), np.uint8), int(valid.sum())
    return np.concatenate(pos_out), np.concatenate(col_out), int(valid.sum())


def weld(pos, col):
    """merge: one vertex per distinct float position (a dict, as std::map<tuple<float,float,float>, int>), ids and colours by first
    appearance over the face corners."""
    ids, verts, cols = {}, [], []
    faces = np.empty(pos.shape[:2], np.int32)
    for f in range(pos.shape[0]):
        for k in range(3):
            key = tuple(float(a) for a in pos[f, k])
            i = ids.get(key)
            if i is None:
                i = ids[key] = len(verts)
                verts.append(pos[f, k])
                cols.append(col[f, k])
            faces[f, k] = i
    V = np.array(verts, F32).reshape(-1, 3)
    C = np.array(cols, np.uint8).reshape(-1, 3)
    return V, C, faces


def clean(verts, faces):
    """removeDegenerateFaces: repeated indices, or a float32 cross product (v2 - v0) x (v2 - v1) with squared norm 0, NaN or Inf."""
    if len(faces) == 0:
        return faces
    a, b, c = faces[:, 0], faces[:, 1], faces[:, 2]
    e0 = verts[c] - verts[a]
    e1 = verts[c] - verts[b]
    cx = e0[:, 1] * e1[:, 2] - e0[:, 2] * e1[:, 1]
    cy = e0[:, 2] * e1[:, 0] - e0[:, 0] * e1[:, 2]
    cz = e0[:, 0] * e1[:, 1] - e0[:, 1] * e1[:, 0]
    with np.errstate(over="ignore", invalid="ignore"):
        sq = (cx * cx + cy * cy) + cz * cz
    keep = (a != b) & (a != c) & (b != c) & (sq != 0) & np.isfinite(sq)
    return faces[keep]


def largest_component(verts, cols, faces):
    """removeLooseComponents + removeUnusedVertices: faces sharing a vertex are connected; the component with the most faces wins, ties
    to the one holding the lowest face index; then the unused vertices go, in order."""
    if len(faces) == 0:
        return verts[:0], cols[:0], faces
    V = len(verts)
    r = np.concatenate([faces[:, 0], faces[:, 0]])
    c = np.concatenate([faces[:, 1], faces[:, 2]])
    _, lab = connected_components(coo_matrix((np.ones(len(r)), (r, c)), shape=(V, V)), directed=False)
    flab = lab[faces[:, 0]]
    count = np.bincount(flab, minlength=lab.max() + 1)
    first = np.full(len(count), len(faces))
    np.minimum.at(first, flab, np.arange(len(faces)))
    best = min(range(len(count)), key=lambda k: (-count[k], first[k]))
    faces = faces[flab == best]
    used = np.zeros(V, bool)
    used[faces.ravel()] = True
    new_id = np.cumsum(used) - 1
    return verts[used], cols[used], new_id[faces].astype(np.int32)


def extract(xyz, sdf, weight, rgb, voxel_size, largest_component_only=False):
    """The whole chain; returns the dict Engine.extract_mesh returns, with info as a dict of the counts."""
    pos, col, cubes = marching_cubes(xyz, sdf, weight, rgb, voxel_size)
    V, C, faces = weld(pos, col)
    fc = clean(V, faces)
    info = dict(num_cubes=cubes, num_faces_raw=len(pos), num_vertices_welded=len(V), num_faces_clean=len(fc))
    if largest_component_only:
        V, C, fc = largest_component(V, C, fc)
    info.update(num_faces=len(fc), num_vertices=len(V))
    return dict(vertices=V, colors=C, faces=fc.astype(np.int32).reshape(-1, 3), info=info)


def extract_grid(g, source="refined", largest_component_only=False):
    """extract() of a grid dict as Engine.download_grid returns it (xyz, sdf0, sdf_refined, weight, rgb, voxel_size)."""
    sdf = g["sdf_refined"] if source == "refined" else g["sdf0"]
    return extract(g["xyz"], sdf, g["weight"], g["rgb"], g["voxel_size"], largest_component_only)
