"""CPU tests of the mesh simplification's numpy restatement tests/mesh_simplify_ref.py (the checker of the k_simp_* kernels): known
answers on constructed meshes, the Jacobi eigen-decomposition against numpy.linalg.eigh, the quality on the bumpy sphere over
tests/mesh_ref.py extractions, and the golden fixture."""
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

import mesh_ref
import mesh_simplify_ref as msr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MESH = ("vertices", "colors", "faces")


def grid_mesh(n, f):
    """An n x n vertex grid triangulated into 2 (n-1)^2 faces, vertex (i, j) at f(i, j) -> xyz; colours by index."""
    ij = np.array([(i, j) for j in range(n) for i in range(n)], np.float64)
    v = np.array([f(i, j) for i, j in ij], np.float32)
    faces = []
    for j in range(n - 1):
        for i in range(n - 1):
            a, b, c, d = j * n + i, j * n + i + 1, (j + 1) * n + i, (j + 1) * n + i + 1
            faces += [(a, b, d), (a, d, c)]
    col = (np.arange(3 * len(v)).reshape(-1, 3) * 29 % 256).astype(np.uint8)
    return dict(vertices=v, colors=col, faces=np.array(faces, np.int32))


def box_mesh(lo, hi, n):
    """The closed surface of the box [lo, hi]^3, each side an n x n vertex grid (welded along the edges), outward faces."""
    t = np.linspace(lo, hi, n)
    verts, index, faces = [], {}, []

    def vid(p):
        key = tuple(np.float32(p))
        if key not in index:
            index[key] = len(verts)
            verts.append(key)
        return index[key]

    for axis in range(3):
        for side, sign in ((lo, -1), (hi, 1)):
            u, w = [a for a in range(3) if a != axis]
            ids = np.empty((n, n), np.int64)
            for i in range(n):
                for j in range(n):
                    p = np.zeros(3)
                    p[axis], p[u], p[w] = side, t[i], t[j]
                    ids[i, j] = vid(p)
            for i in range(n - 1):
                for j in range(n - 1):
                    a, b, c, d = ids[i, j], ids[i + 1, j], ids[i + 1, j + 1], ids[i, j + 1]
                    tri = [(a, b, c), (a, c, d)]
                    # orient outwards: (p_b - p_a) x (p_c - p_a) along sign * e_axis
                    pa, pb, pc = (np.array(verts[k], np.float64) for k in (a, b, c))
                    if np.cross(pb - pa, pc - pa)[axis] * sign < 0:
                        tri = [(x, z, y) for x, y, z in tri]
                    faces += tri
    v = np.array(verts, np.float32)
    return dict(vertices=v, colors=np.full((len(v), 3), 200, np.uint8), faces=np.array(faces, np.int32))


def sphere_mesh(largest_component_only=True):
    import test_mesh as tm
    xyz, sdf, w, rgb = tm.grid(tm._sphere((3.3, 2.6, 4.1), 2.2, half=4))
    return mesh_ref.extract(xyz, sdf, w, rgb, 0.004, largest_component_only)


def min_chebyshev_spacing(v):
    d, _ = cKDTree(v.astype(np.float64)).query(v.astype(np.float64), k=2, p=np.inf)
    return float(d[:, 1].min())


# ---- known answers ------------------------------------------------------------------------------------------------------------------
def test_tilted_plane_stays_on_plane():
    a, b, c = 0.3, -0.2, 0.7
    rng = np.random.default_rng(3)
    jit = rng.uniform(-0.3, 0.3, (40, 40, 2))

    def f(i, j):
        x, y = 0.01 * (i + jit[int(i), int(j), 0]), 0.01 * (j + jit[int(i), int(j), 1])
        return (x, y, a * x + b * y + c)

    m = grid_mesh(40, f)
    for cell in (0.02, 0.05, 0.1):
        s = msr.simplify(m, cell)
        v = s["vertices"].astype(np.float64)
        assert len(s["faces"]) < len(m["faces"]) and len(v) > 3
        off = np.abs(v[:, 2] - (a * v[:, 0] + b * v[:, 1] + c))
        assert off.max() <= 4 * np.spacing(np.float32(c + 0.3)), (cell, off.max())
        print(cell, len(m["faces"]), "->", len(s["faces"]), "max off-plane", off.max())


def test_cube_corners_reproduced():
    """Cells of 0.5 m around a box from 0.05 to 0.95 m: each corner cell holds one box corner and parts of its three sides, whose
    planes meet exactly there.  The mean of the cell's vertices lies well inside the box."""
    m = box_mesh(0.05, 0.95, 4)
    s = msr.simplify(m, 0.5)
    corners = np.array([(x, y, z) for x in (0.05, 0.95) for y in (0.05, 0.95) for z in (0.05, 0.95)], np.float32).astype(np.float64)
    v = s["vertices"].astype(np.float64)
    assert len(v) == 8 and len(s["faces"]) == 12
    for p in v:
        assert np.abs(corners - p).max(1).min() <= 2 * np.spacing(np.float32(0.95)), p
    # clustering by the mean would put the corner cells' vertices inside the box
    cl = msr.cells(m["vertices"], 0.5)
    mean0 = m["vertices"][(cl == 0).all(1)].astype(np.float64).mean(0)
    assert np.abs(mean0 - 0.05).min() > 0.05


def test_tiny_cell_is_identity():
    m = sphere_mesh()
    assert len(m["faces"]) > 100
    cell = 0.5 * min_chebyshev_spacing(m["vertices"])
    s = msr.simplify(m, cell)
    for k in MESH:
        assert s[k].tobytes() == m[k].tobytes(), k
    assert s["info"]["num_clusters"] == len(m["vertices"])
    assert s["info"]["num_faces_collapsed"] == s["info"]["num_faces_duplicate"] == s["info"]["num_faces_degenerate"] == 0


def test_whole_mesh_cell_is_empty():
    m = sphere_mesh()
    assert (m["vertices"] > 0).all() and (m["vertices"] < 1).all()
    s = msr.simplify(m, 1.0)
    assert s["info"]["num_clusters"] == 1 and s["info"]["num_faces_collapsed"] == len(m["faces"])
    assert s["vertices"].shape == (0, 3) and s["colors"].shape == (0, 3) and s["faces"].shape == (0, 3)
    from intrinsic3d_b200.mesh import save_ply
    with pytest.raises(ValueError):
        save_ply(os.devnull, s)


def test_refuses_cells_outside_int32():
    m = sphere_mesh()
    for cell in (1e-12, float("nan")):
        with pytest.raises(ValueError):
            msr.simplify(m, cell)


def test_duplicates_and_orientation():
    """Two faces on the same three clusters in the same orientation: the later one is a duplicate; the opposite orientation stays."""
    v = np.array([(0.1, 0.1, 0.1), (1.1, 0.1, 0.1), (0.1, 1.1, 0.1), (0.12, 0.1, 0.1), (1.12, 0.1, 0.1), (0.1, 1.12, 0.1)], np.float32)
    m = dict(vertices=v, colors=np.zeros((6, 3), np.uint8), faces=np.array([(0, 1, 2), (4, 5, 3), (3, 5, 4), (0, 1, 3)], np.int32))
    s = msr.simplify(m, 0.5)
    assert s["info"]["num_clusters"] == 3
    assert s["info"]["num_faces_collapsed"] == 1 and s["info"]["num_faces_duplicate"] == 1
    assert s["faces"].tolist() == [[0, 1, 2], [0, 2, 1]]


# ---- the eigen-decomposition ----------------------------------------------------------------------------------------------------------
def _check_eigen(a):
    lam, vec = msr.jacobi3(a)
    for k in range(len(a)):
        ref = np.linalg.eigh(a[k])[0]
        scale = max(1.0, np.abs(ref).max())
        assert np.abs(np.sort(lam[k]) - ref).max() <= 1e-12 * scale, (a[k], lam[k], ref)
        assert np.abs(vec[k].T @ vec[k] - np.eye(3)).max() <= 1e-12
        assert np.abs(a[k] @ vec[k] - vec[k] * lam[k]).max() <= 1e-12 * scale


def test_jacobi_matches_eigh():
    rng = np.random.default_rng(11)
    g = rng.normal(size=(500, 3, 3))
    _check_eigen(g @ np.swapaxes(g, 1, 2) + 1e-3 * np.eye(3))          # SPD
    for rank in (1, 2):
        u = rng.normal(size=(500, 3, rank))
        _check_eigen(u @ np.swapaxes(u, 1, 2))
    _check_eigen(np.stack([np.diag([3.0, 1.0, 2.0]), np.zeros((3, 3))]))   # already diagonal: every rotation skipped


# ---- quality on the bumpy sphere --------------------------------------------------------------------------------------------------------
# Bounds from the measured values (this restatement, which the device reproduces byte for byte), rounded up: the largest radial
# distance |r - rho(d)| of an output vertex from the analytic surface, in voxels, and the output / input face ratio.  Measured, the
# fused sdf, largest component (input: 3792 / 15456 faces, vertices at most 0.231 / 0.225 voxels off the surface):
#   tiny  2 voxels: 820 faces (0.216), max 0.213, mean 0.042     tiny  4 voxels: 230 faces (0.061), max 0.272, mean 0.087
#   small 2 voxels: 3377 faces (0.218), max 0.189, mean 0.038    small 4 voxels: 908 faces (0.059), max 0.223, mean 0.059
QUALITY = {
    ("tiny", 2): (0.22, 0.22),
    ("tiny", 4): (0.28, 0.062),
    ("small", 2): (0.19, 0.22),
    ("small", 4): (0.23, 0.06),
}


@pytest.mark.parametrize("scene,factor", sorted(QUALITY))
def test_bumpy_sphere_quality(scene, factor, request):
    import torch
    from intrinsic3d_b200 import scene as sc
    s = request.getfixturevalue(f"{scene}_scene")
    vs = float(s["voxel_size"])
    m = mesh_ref.extract(s["xyz"], s["sdf0"], s["weight"], s["rgb"], vs, True)
    out = msr.simplify(m, factor * vs)
    radius = {"tiny": 10.0, "small": 20.0}[scene] * float(np.float32(vs))

    def dist(v):
        return np.abs(sc._implicit(torch.tensor(v, dtype=torch.float64), torch.zeros(3, dtype=torch.float64), radius, 0.03).numpy()) / vs

    d_in, d_out = dist(m["vertices"]), dist(out["vertices"])
    ratio = len(out["faces"]) / len(m["faces"])
    print(scene, factor, len(m["faces"]), "->", len(out["faces"]), f"ratio {ratio:.4f}", f"input max {d_in.max():.4f} vox",
          f"output max {d_out.max():.4f} mean {d_out.mean():.4f} vox")
    max_dist, max_ratio = QUALITY[(scene, factor)]
    assert d_out.max() <= max_dist and ratio <= max_ratio


# ---- the fixture -------------------------------------------------------------------------------------------------------------------
def test_golden_fixture_matches_restatement():
    g = np.load(os.path.join(ROOT, "tests", "golden", "tiny_mesh_simplify.npz"))
    src = dict(vertices=g["in_vertices"], colors=g["in_colors"], faces=g["in_faces"])
    prev = None
    for k, cell in enumerate(g["cells"]):
        s = msr.simplify(prev if g["chained"][k] else src, float(cell))
        for key in MESH:
            assert s[key].tobytes() == g[f"{k}_{key}"].tobytes(), (k, key)
        assert [s["info"][c] for c in msr.INFO_COUNTS] == g[f"{k}_info"].tolist()
        prev = s
