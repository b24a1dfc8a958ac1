"""CPU tests of the surface extraction: the generated case tables, the numpy restatement tests/mesh_ref.py (the checker of the
kernels) on constructed grids, and the PLY writer."""
import ctypes as C
import itertools
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "intrinsic3d_b200", "csrc"))
import gen_mc_tables  # noqa: E402
import mesh_ref  # noqa: E402

REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libmc_ref_tables.so")


def grid(values, weight=None, rgb=None, drop=()):
    """Grid arrays from {coords: sdf}; voxels in the dict's order."""
    xyz = np.array([k for k in values if k not in drop], np.int32).reshape(-1, 3)
    sdf = np.array([values[tuple(k)] for k in xyz], np.float64)
    w = np.ones(len(xyz), np.float32) if weight is None else np.array([weight.get(tuple(k), 1.0) for k in xyz], np.float32)
    col = (np.arange(3 * len(xyz)).reshape(-1, 3) * 37 % 256).astype(np.uint8) if rgb is None else rgb
    return xyz, sdf, w, col


def cube(case, lo=-1.0, hi=1.0, origin=(0, 0, 0)):
    """The 8 voxels of one cube with the corners of `case` inside (sdf lo) and the rest at hi."""
    vals = {}
    for c, off in enumerate(gen_mc_tables.CORNERS):
        vals[tuple(o + d for o, d in zip(origin, off))] = lo if (case >> c) & 1 else hi
    return vals


def edges_of(faces):
    out = {}
    for f in faces:
        for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])):
            out.setdefault((min(a, b), max(a, b)), []).append((a, b))
    return out


# ---- the generated tables --------------------------------------------------------------------------------------------------------
def test_header_equals_generator():
    path = os.path.join(ROOT, "intrinsic3d_b200", "csrc", "i3d_mc_tables.cuh")
    assert open(path).read() == gen_mc_tables.render()


def test_tables_by_rule():
    masks, tris = gen_mc_tables.tables()
    assert sum(len(t) for t in tris) == 820
    for case in range(256):
        inside = [(case >> c) & 1 for c in range(8)]
        crossing = {e for e, (a, b) in enumerate(gen_mc_tables.EDGES) if inside[a] != inside[b]}
        assert masks[case] == sum(1 << e for e in crossing)
        assert {e for t in tris[case] for e in t} == crossing     # every crossing edge is used, no other
        assert masks[255 - case] == masks[case]


def _boundary(tris):
    """Directed boundary edges of a triangle set (interior diagonals cancel against their reverse)."""
    cnt = {}
    for t in tris:
        for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            if cnt.get((b, a), 0) > 0:
                cnt[(b, a)] -= 1
            else:
                cnt[(a, b)] = cnt.get((a, b), 0) + 1
    return sorted(k for k, v in cnt.items() for _ in range(v))


@pytest.mark.skipif(not os.path.exists(REF_LIB), reason="oracle/_ref/libmc_ref_tables.so not built (needs the reference tree at build time)")
def test_tables_match_reference_polygons():
    L = C.CDLL(REF_LIB)
    et = list((C.c_int * 256).in_dll(L, "i3d_ref_edge_table"))
    tt = list((C.c_int * 4096).in_dll(L, "i3d_ref_triangle_table"))
    masks, tris = gen_mc_tables.tables()
    for case in range(256):
        row = tt[16 * case:16 * case + 16]
        ref = [tuple(row[i:i + 3]) for i in range(0, 16, 3) if row[i] != -1]
        assert et[case] == masks[case], case
        assert len(ref) == len(tris[case]), case
        assert _boundary(ref) == _boundary(tris[case]), case


# ---- single cubes ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(256))
def test_single_cube_case(case):
    xyz, sdf, w, rgb = grid(cube(case))
    m = mesh_ref.extract(xyz, sdf, w, rgb, 1.0)
    masks, tris = gen_mc_tables.tables()
    assert m["info"]["num_cubes"] == 1
    assert len(m["faces"]) == len(tris[case])
    # sdf -1 / +1: every vertex is an edge midpoint, one per crossing edge
    mids = {tuple((np.array(gen_mc_tables.CORNERS[a]) + gen_mc_tables.CORNERS[b]) / 2.0)
            for e, (a, b) in enumerate(gen_mc_tables.EDGES) if masks[case] >> e & 1}
    assert {tuple(v) for v in m["vertices"].astype(np.float64)} == mids
    # right-hand normals point towards sdf >= 0: the normal's component along each vertex's edge, inside -> outside, is never negative
    # summed over a triangle (zero for a fan triangle standing across a saddle), and positive summed over the case
    V = m["vertices"].astype(np.float64)
    inside = [(case >> c) & 1 for c in range(8)]
    total = 0.0
    for f in m["faces"]:
        nrm = np.cross(V[f[1]] - V[f[0]], V[f[2]] - V[f[0]])
        s = 0.0
        for k in f:
            for a, b in gen_mc_tables.EDGES:
                if inside[a] != inside[b] and np.allclose((np.array(gen_mc_tables.CORNERS[a]) + gen_mc_tables.CORNERS[b]) / 2.0, V[k]):
                    ci, co = (a, b) if inside[a] else (b, a)
                    s += nrm @ (np.array(gen_mc_tables.CORNERS[co]) - gen_mc_tables.CORNERS[ci])
        assert s >= 0, (case, f)
        total += s
    assert case in (0, 255) or total > 0, case


def _sphere(center, radius, half=6):
    c = np.array(center, np.float64)
    base = np.floor(c).astype(int)
    vals = {}
    for d in itertools.product(range(-half, half + 1), repeat=3):
        p = base + np.array(d)
        vals[tuple(int(v) for v in p)] = float(np.linalg.norm(p - c) - radius)
    return vals


def test_sphere_closed_and_outward():
    # far from the origin (coordinates ~ 2^16, voxel size 1): the float positions of one lattice edge interpolated from either end agree
    c = (70000.37, 70000.61, 70000.23)
    xyz, sdf, w, rgb = grid(_sphere(c, 4.3))
    assert np.abs(sdf).min() > 1e-3
    m = mesh_ref.extract(xyz, sdf, w, rgb, 1.0)
    F, V = m["faces"], m["vertices"].astype(np.float64)
    assert m["info"]["num_faces_clean"] == m["info"]["num_faces_raw"]
    E = edges_of(F)
    assert all(len(v) == 2 for v in E.values())
    assert all(v[0] != v[1] for v in E.values())          # consistently oriented: each edge once in each direction
    assert len(V) - len(E) + len(F) == 2
    cen = np.array(c)
    for f in F:
        nrm = np.cross(V[f[1]] - V[f[0]], V[f[2]] - V[f[0]])
        assert nrm @ (V[f].mean(0) - cen) > 0
    # one component: the filter changes nothing
    m2 = mesh_ref.extract(xyz, sdf, w, rgb, 1.0, largest_component_only=True)
    for k in ("vertices", "colors", "faces"):
        assert m2[k].tobytes() == m[k].tobytes()


@pytest.mark.parametrize("zero", [0.0, 5e-6, -0.0])
def test_near_zero_corner_welds_and_drops_degenerate(zero):
    # inside c0, c2, c3 of the bottom face, c1 (outside) at ~0: edges e0 and e1 both return c1's position -> one vertex, and the fan
    # triangle holding both is degenerate
    vals = cube(1 | 4 | 8)
    vals[gen_mc_tables.CORNERS[1]] = zero
    xyz, sdf, w, rgb = grid(vals)
    m = mesh_ref.extract(xyz, sdf, w, rgb, 1.0)
    info = m["info"]
    assert info["num_faces_raw"] == 3
    assert info["num_vertices_welded"] == 4                 # 5 crossing edges, two of them at c1
    assert info["num_faces_clean"] == 2
    assert np.array([1, 0, 0], np.float32).tobytes() in {v.tobytes() for v in m["vertices"]}


def test_unused_vertex_kept_without_filter():
    # only c4 outside, at sdf 0: the single triangle collapses onto c4 and is dropped; its vertex stays unless the filter runs
    vals = cube(255 - 16)
    vals[gen_mc_tables.CORNERS[4]] = 0.0
    xyz, sdf, w, rgb = grid(vals)
    m = mesh_ref.extract(xyz, sdf, w, rgb, 1.0)
    assert m["info"]["num_faces_raw"] == 1 and len(m["faces"]) == 0 and len(m["vertices"]) == 1
    m2 = mesh_ref.extract(xyz, sdf, w, rgb, 1.0, largest_component_only=True)
    assert len(m2["faces"]) == 0 and len(m2["vertices"]) == 0


def opposite_end_grid():
    """Two cubes side by side (x = 0..2) with sdf depending on y only, at values for which the shared lattice edges give different
    floats from the two ends (Q42): every y-edge crosses, the two at x = 1 are interpolated from opposite ends."""
    rng = np.random.default_rng(0)
    for _ in range(10000):
        sa, sb = -float(np.float32(rng.uniform(0.01, 1))), float(np.float32(rng.uniform(0.01, 1)))
        f = np.float32
        # cube 0, e0: from y = 1 (sb) to y = 0 (sa); cube 1, e2: from y = 0 (sa) to y = 1 (sb)
        mu0 = (f(0) - f(sb)) / (f(sa) - f(sb))
        mu1 = (f(0) - f(sa)) / (f(sb) - f(sa))
        y0 = f(1) + mu0 * (f(0) - f(1))
        y1 = f(0) + mu1 * (f(1) - f(0))
        if y0 != y1:
            break
    else:
        raise AssertionError("no opposite-end pair found")
    vals = {(x, y, z): (sa if y == 0 else sb) for z in (0, 1) for y in (0, 1) for x in (0, 1, 2)}
    return grid(vals)


def test_opposite_ends_keep_two_vertices():
    xyz, sdf, w, rgb = opposite_end_grid()
    m = mesh_ref.extract(xyz, sdf, w, rgb, 1.0)
    assert m["info"]["num_cubes"] == 2
    assert len(m["faces"]) == 4
    assert len(m["vertices"]) == 8                         # 6 lattice edges cross; the 2 shared ones give 2 vertices each


def test_missing_or_zero_weight_corner_skips_cube():
    vals = cube(1)
    c111 = gen_mc_tables.CORNERS[4]
    m = mesh_ref.extract(*grid(vals, drop=(c111,)), 1.0)
    assert m["info"]["num_cubes"] == 0 and len(m["faces"]) == 0
    for c in range(8):
        m = mesh_ref.extract(*grid(vals, weight={gen_mc_tables.CORNERS[c]: 0.0}), 1.0)
        assert m["info"]["num_cubes"] == 0 and len(m["faces"]) == 0


def two_blobs(first_tris, second_tris):
    """Two separate cubes far apart; the first in voxel order has `first_tris` triangles (1 or 2), the second `second_tris`."""
    case = {1: 1, 2: 1 | 2}
    vals = dict(cube(case[first_tris], origin=(40, 0, 0)))
    vals.update(cube(case[second_tris], origin=(0, 0, 0)))
    return grid(vals)


def test_floaters_removed_and_tie_rule():
    m = mesh_ref.extract(*two_blobs(1, 2), 1.0, largest_component_only=True)
    assert len(m["faces"]) == 2 and len(m["vertices"]) == 4
    assert (m["vertices"][:, 0] < 10).all()                # the 2-triangle blob, second in voxel order
    # a tie: the component that holds face 0 (the cube first in voxel order, here the one at x = 40) wins
    m = mesh_ref.extract(*two_blobs(1, 1), 1.0, largest_component_only=True)
    assert len(m["faces"]) == 1 and (m["vertices"][:, 0] > 10).all()
    assert m["faces"].tolist() == [[0, 1, 2]]


def test_empty_result():
    xyz, sdf, w, rgb = grid(cube(0))
    for lc in (False, True):
        m = mesh_ref.extract(xyz, sdf, w, rgb, 1.0, lc)
        assert m["vertices"].shape == (0, 3) and m["colors"].shape == (0, 3) and m["faces"].shape == (0, 3)
    from intrinsic3d_b200.mesh import save_ply
    with pytest.raises(ValueError):
        save_ply(os.devnull, m)


# ---- PLY ----------------------------------------------------------------------------------------------------------------------------
def _parse_ply(data):
    """An independent reader of the binary little-endian PLY that Mesh::save writes."""
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").split("\n")
    assert header[0] == "ply" and header[1] == "format binary_little_endian 1.0"
    nv = int(header[2].split()[2])
    assert header[3:9] == ["property float x", "property float y", "property float z", "property uchar red", "property uchar green",
                           "property uchar blue"]
    nf = int(header[9].split()[2])
    assert header[10:] == ["property list uchar int vertex_indices", "end_header", ""]
    off, verts, cols, faces = end, [], [], []
    for _ in range(nv):
        x, y, z, r, g, b = struct.unpack_from("<fffBBB", data, off)
        off += 15
        verts.append((x, y, z))
        cols.append((r, g, b))
    for _ in range(nf):
        k, a, b, c = struct.unpack_from("<Biii", data, off)
        assert k == 3
        off += 13
        faces.append((a, b, c))
    assert off == len(data)
    return np.array(verts, np.float32).reshape(-1, 3), np.array(cols, np.uint8).reshape(-1, 3), np.array(faces, np.int32).reshape(-1, 3)


def test_ply_bytes(tmp_path):
    from intrinsic3d_b200.mesh import save_ply
    xyz, sdf, w, rgb = grid(_sphere((3.3, 2.6, 4.1), 2.2, half=4))
    m = mesh_ref.extract(xyz, sdf, w, rgb, 0.004)
    assert len(m["faces"]) > 0
    p = tmp_path / "m.ply"
    save_ply(p, m)
    data = p.read_bytes()
    assert data.startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % len(m["vertices"]))
    assert len(data) == data.index(b"end_header\n") + 11 + 15 * len(m["vertices"]) + 13 * len(m["faces"])
    v, c, f = _parse_ply(data)
    assert v.tobytes() == m["vertices"].tobytes() and c.tobytes() == m["colors"].tobytes() and f.tobytes() == m["faces"].tobytes()
    # a mesh with vertices but no faces is written (Mesh::save only refuses an empty vertex list)
    save_ply(p, dict(vertices=m["vertices"][:2], colors=m["colors"][:2], faces=np.zeros((0, 3), np.int32)))
    v, c, f = _parse_ply(p.read_bytes())
    assert len(v) == 2 and len(f) == 0


def test_golden_fixture_matches_restatement():
    g = np.load(os.path.join(ROOT, "tests", "golden", "tiny_mesh.npz"))
    grid_ = dict(xyz=g["xyz"], sdf0=g["sdf0"], sdf_refined=g["sdf_refined"], weight=g["weight"], rgb=g["rgb"], voxel_size=float(g["voxel_size"]))
    for src in ("fused", "refined"):
        for lc in (0, 1):
            m = mesh_ref.extract_grid(grid_, src, bool(lc))
            tag = f"{src}_{lc}"
            for k in ("vertices", "colors", "faces"):
                assert m[k].tobytes() == g[f"{tag}_{k}"].tobytes(), (tag, k)
