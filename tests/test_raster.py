"""CPU tests of the rasterizer's restatement (tests/raster_ref.py, DESIGN.md §6w): known answers, watertightness, ties, the camera
plane, distortion, the colour rules, the candidate pairs against brute force, and the fixture."""
import os

import numpy as np
import pytest

import raster_ref as ra
import render_ref as rr
import texture_ref as tr

f32 = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))
EYE = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], f32)
CAM = dict(fx=f32(40.0), fy=f32(40.0), cx=f32(15.5), cy=f32(11.5), d=np.zeros(5, f32))
W, H = 32, 24


def _mesh(V, F, colors=None):
    V = np.asarray(V, f32).reshape(-1, 3)
    c = np.full((len(V), 3), 100, np.uint8) if colors is None else np.asarray(colors, np.uint8)
    return dict(vertices=V, faces=np.asarray(F, np.int32).reshape(-1, 3), colors=c)


def _point_in_tri(px, py, tri):
    """exact (float64) containment of points in a 2-D triangle, edges included"""
    (x0, y0), (x1, y1), (x2, y2) = tri
    d1 = (px - x1) * (y0 - y1) - (x0 - x1) * (py - y1)
    d2 = (px - x2) * (y1 - y2) - (x1 - x2) * (py - y2)
    d3 = (px - x0) * (y2 - y0) - (x2 - x0) * (py - y0)
    neg = (d1 < 0) | (d2 < 0) | (d3 < 0)
    pos = (d1 > 0) | (d2 > 0) | (d3 > 0)
    return ~(neg & pos)


def test_fronto_parallel_triangle_known_answer():
    z0 = f32(2.0)
    tri = np.array([[-0.2, -0.15], [0.25, -0.1], [-0.05, 0.2]])
    m = _mesh([[x * z0, y * z0, z0] for x, y in tri], [[0, 1, 2]])
    tri = m["vertices"][:, :2].astype(np.float64) / 2.0             # the float vertices, exactly
    r = ra.rasterize(m, EYE[None], CAM, W, H)
    rx, ry = ra.rays(CAM, W, H)
    inside = _point_in_tri(rx.astype(np.float64), ry.astype(np.float64), tri)
    cov = r["face"][0] == 0
    # exactly the pixels whose rays the triangle contains
    assert cov.tobytes() == inside.tobytes() and cov.sum() > 20
    assert np.all(r["depth"][0][cov] == z0) and np.all(r["depth"][0][~cov] == 0)
    # linear barycentrics: the weights reproduce the ray's position
    a, b = r["bary"][0][cov, 0].astype(np.float64), r["bary"][0][cov, 1].astype(np.float64)
    w0 = 1 - a - b
    x = w0 * tri[0, 0] + a * tri[1, 0] + b * tri[2, 0]
    y = w0 * tri[0, 1] + a * tri[1, 1] + b * tri[2, 1]
    assert np.abs(x - rx[cov]).max() < 1e-5 and np.abs(y - ry[cov]).max() < 1e-5
    n = r["normal"][0][cov]
    assert np.allclose(np.abs(n[:, 2]), 1.0) and np.all(r["normal"][0][~cov] == 0)


def _square(z, s=0.5):
    return [[-s * z, -s * z, z], [s * z, -s * z, z], [s * z, s * z, z], [-s * z, s * z, z]]


def test_nearer_wins_and_ties_go_to_the_lowest_face():
    V = _square(3.0) + _square(2.0)
    m = _mesh(V, [[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]])
    r = ra.rasterize(m, EYE[None], CAM, W, H)
    cov = r["face"][0] >= 0
    assert cov.all() and np.all(np.isin(r["face"][0], [2, 3])) and np.all(r["depth"][0] == f32(2.0))
    # coplanar duplicates, either orientation: the lowest id wins
    m = _mesh(_square(2.0), [[0, 2, 1], [0, 1, 2], [0, 3, 2], [0, 2, 3]])
    r = ra.rasterize(m, EYE[None], CAM, W, H)
    assert set(np.unique(r["face"][0])) <= {0, 2}


def test_faces_behind_and_straddling_the_camera_plane():
    behind = _mesh([[-1, -1, -1], [1, -1, -1], [0, 1, -1]], [[0, 1, 2]])
    assert np.all(ra.rasterize(behind, EYE[None], CAM, W, H)["face"] == -1)
    # a face through the camera plane: only its part in front is hit, at positive depth, where the ray meets its plane
    st = _mesh([[-2, -2, -1], [2, -2, -1], [0, 3, 4]], [[0, 1, 2]])
    r = ra.rasterize(st, EYE[None], CAM, W, H)
    rb = ra.rasterize(st, EYE[None], CAM, W, H, brute=True)
    cov = r["face"][0] == 0
    assert cov.sum() > 0 and np.all(r["depth"][0][cov] > 0)
    assert all(r[k].tobytes() == rb[k].tobytes() for k in ra.PLANES)
    # the plane through the vertices: z = 1 + y (y up the face), so depth = 1 / (1 - y_ray)
    rx, ry = ra.rays(CAM, W, H)
    assert np.allclose(r["depth"][0][cov], 1.0 / (1.0 - ry[cov].astype(np.float64)), rtol=1e-5)


def test_distortion_coverage_follows_the_undistorted_rays():
    cam = dict(CAM, d=np.array([0.08, -0.02, 0.004, 0.003, -0.002], f32))
    tri = np.array([[-0.3, -0.25], [0.35, -0.2], [0.0, 0.3]])
    m = _mesh([[x * 2, y * 2, 2] for x, y in tri], [[0, 1, 2]])
    tri = m["vertices"][:, :2].astype(np.float64) / 2.0
    r = ra.rasterize(m, EYE[None], cam, W, H)
    rx, ry = ra.rays(cam, W, H)
    inside = _point_in_tri(rx.astype(np.float64), ry.astype(np.float64), tri)
    cov = r["face"][0] == 0
    assert cov.tobytes() == inside.tobytes()
    assert cov.tobytes() != (ra.rasterize(m, EYE[None], CAM, W, H)["face"][0] == 0).tobytes()
    assert all(r[k].tobytes() == ra.rasterize(m, EYE[None], cam, W, H, brute=True)[k].tobytes() for k in ra.PLANES)


@pytest.mark.parametrize("oblique", [False, True])
def test_watertight_grid_through_pixel_rays(oblique):
    """A planar grid of triangles with shared float vertices, with pixel rays through its vertices and edges: every pixel whose ray
    meets the plane inside the outline is covered."""
    cam = dict(fx=f32(8.0), fy=f32(8.0), cx=f32(15.0), cy=f32(11.0), d=np.zeros(5, f32))
    z = f32(2.0)
    n = 6
    g = np.linspace(-1.0, 1.0, n + 1).astype(f32)         # vertices at x, y = k / 3 -> rays of pixels u = cx + 8 k / 3 ...
    g = (np.round(g * 4) / 4).astype(f32)                  # quarter steps: pixel rays (u - cx) / 8 hit every vertex and edge
    X, Y = np.meshgrid(g, g)
    V = np.stack([X.ravel() * z, Y.ravel() * z, np.full(X.size, z)], 1).astype(f32)
    if oblique:
        V[:, 2] = (z + f32(0.25) * V[:, 0] / z).astype(f32)          # tilt: z = 2 + x / 8 on the vertices
        V[:, 0] = (g[np.arange(X.size) % (n + 1)] * V[:, 2]).astype(f32)
        V[:, 1] = (g[np.arange(X.size) // (n + 1)] * V[:, 2]).astype(f32)
    F = []
    for j in range(n):
        for i in range(n):
            a, b, c, d = j * (n + 1) + i, j * (n + 1) + i + 1, (j + 1) * (n + 1) + i + 1, (j + 1) * (n + 1) + i
            F += [[a, b, c], [a, c, d]] if (i + j) % 2 else [[a, b, d], [b, c, d]]
    m = _mesh(V, F)
    r = ra.rasterize(m, EYE[None], cam, W, H)
    rx, ry = ra.rays(cam, W, H)
    lo, hi = float(g.min()), float(g.max())
    inside = (rx >= lo) & (rx <= hi) & (ry >= lo) & (ry <= hi)
    cov = r["face"][0] >= 0
    assert np.all(cov[inside]), "a crack"
    assert not np.any(cov[~inside])
    assert all(r[k].tobytes() == ra.rasterize(m, EYE[None], cam, W, H, brute=True)[k].tobytes() for k in ra.PLANES)


def test_vertex_colour_rules():
    z = f32(2.0)
    tri = np.array([[-0.3, -0.2], [0.3, -0.2], [0.0, 0.25]])
    V = [[x * z, y * z, z] for x, y in tri]
    cols = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255]], np.uint8)
    r = ra.rasterize(_mesh(V, [[0, 1, 2]], cols), EYE[None], CAM, W, H, color="vertex")
    cov = r["face"][0] == 0
    a, b = r["bary"][0][cov, 0], r["bary"][0][cov, 1]
    rgb = r["rgb"][0][cov].astype(np.float64)
    assert np.abs(rgb - 255 * np.stack([1 - a - b, a, b], 1)).max() <= 1.0
    # at a vertex (a = b = 0): that vertex's colour
    hit, t, a, b = ra.hit(np.array([[V[0], V[1], V[2]]], f32), np.array([tri[0, 0]], f32), np.array([tri[0, 1]], f32))
    assert hit[0] and a[0] == 0 and b[0] == 0
    r = ra.rasterize(_mesh(V, [[0, 1, 2]], np.full((3, 3), 77, np.uint8)), EYE[None], CAM, W, H, color="vertex")
    assert np.all(r["rgb"][0][cov] == 77) and np.all(r["rgb"][0][~cov] == 0)


@pytest.mark.parametrize("S", [6, 12])
def test_constant_atlas_gives_the_constant_and_reads_owned_texels(S):
    rng = np.random.default_rng(S)
    V = rng.uniform(-0.5, 0.5, (30, 3)).astype(f32)
    V[:, 2] += f32(2.5)
    F = rng.integers(0, 30, (40, 3)).astype(np.int32)
    F = F[(F[:, 0] != F[:, 1]) & (F[:, 1] != F[:, 2]) & (F[:, 0] != F[:, 2])]
    L = tr.layout(len(F), S)
    img = np.full((L["H"], L["W"], 3), (10, 200, 33), np.uint8)
    r = ra.rasterize(_mesh(V, F), EYE[None], CAM, W, H, color="texture", texture=(img, S))   # asserts owned-texel reads
    cov = r["face"][0] >= 0
    # interp_u8 sums the taps and their weights in different orders and truncates, so a constant atlas reads back as c or c - 1
    d = np.array([10, 200, 33]) - r["rgb"][0][cov].astype(np.int64)
    assert cov.sum() > 50 and np.all((d == 0) | (d == 1)) and np.mean(d == 0) > 0.5
    # a random atlas: still only owned texels
    img = rng.integers(0, 256, img.shape).astype(np.uint8)
    ra.rasterize(_mesh(V, F), EYE[None], CAM, W, H, color="texture", texture=(img, S))


def _tiny_mesh():
    import mesh_ref
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("tiny")
    return s, mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], s["rgb"], float(s["voxel_size"]), True)


def test_candidate_pairs_equal_brute_force():
    s, m = _tiny_mesh()
    rts = rr.pose_rt(s["poses"])
    cam = rr.camera(s["intr"], s["dist"])
    cam_d = dict(cam, d=np.array([0.03, -0.01, 0.004, 0.002, -0.0015], f32))
    sub = dict(m, faces=m["faces"][::7])
    for c in (cam, cam_d):
        a = ra.rasterize(sub, rts[:1], c, 160, 120, color="vertex")
        b = ra.rasterize(sub, rts[:1], c, 160, 120, color="vertex", brute=True)
        assert a["face"].max() >= 0
        assert all(a[k].tobytes() == b[k].tobytes() for k in ra.PLANES)
        assert a["tests"] < b["tests"]


def test_fixture():
    s, m = _tiny_mesh()
    z = np.load(os.path.join(HERE, "golden", "tiny_raster.npz"))
    assert z["faces"].tobytes() == m["faces"].astype(np.int32).tobytes()
    from intrinsic3d_b200.scene import make_color_frames
    col = make_color_frames(s)
    ids = z["ids"]
    r = ra.rasterize(m, rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"]), s["depth"].shape[2], s["depth"].shape[1], color="vertex",
                     depth=s["depth"], bgr=col, ids=ids)
    for k in ra.PLANES:
        assert r[k].tobytes() == z[k].tobytes(), k
    got = np.array([[st["num_covered"], st["num_observed"], st["depth_count"], st["color_count"], *st["color_abs"], *st["color_sq"]]
                    for st in r["stats"]], np.int64)
    assert got.tobytes() == z["counts"].tobytes()
    assert np.allclose([[st["depth_abs"], st["depth_sq"]] for st in r["stats"]], z["sums"], rtol=1e-12, atol=0)


def test_faces_in_the_camera_plane_never_hit_wide_rays():
    """A face with every camera z <= 0 is a miss even for rays wider than 45 degrees, where the shear runs along x or y and the sign of
    T no longer follows z: binning, which drops such faces, and brute force agree."""
    rng = np.random.default_rng(7)
    m = 4000
    q = rng.uniform(-1, 1, (m, 3, 3)).astype(f32)
    q[:, :, 2] = np.where(rng.random((m, 1)) < 0.5, f32(-0.0), -rng.uniform(0, 1e-3, (m, 3))).astype(f32)
    x = (rng.uniform(1, 3, m) * rng.choice([-1, 1], m)).astype(f32)
    y = rng.uniform(-3, 3, m).astype(f32)
    assert not ra.hit(q, x, y)[0].any()
    cam = dict(fx=f32(5.0), fy=f32(5.0), cx=f32(15.5), cy=f32(11.5), d=np.zeros(5, f32))          # |x| up to 3.1
    V = np.array([[-3, -2, -0.0], [3, -2, -0.0], [0, 3, -0.0], [-1, -1, 2], [1, -1, 2], [0, 1, 2]], f32)
    msh = _mesh(V, [[0, 1, 2], [3, 4, 5]])
    a, b = ra.rasterize(msh, EYE[None], cam, W, H), ra.rasterize(msh, EYE[None], cam, W, H, brute=True)
    assert all(a[k].tobytes() == b[k].tobytes() for k in ra.PLANES) and set(np.unique(a["face"])) == {-1, 1}


# Measured: the fused tiny mesh against render_ref's march of sdf0, keyframes 0 and 3: median |dz| 0.013 / 0.014 voxel, p99 0.145 /
# 0.139 voxel, and 12 / 15 of ~6 250 pixels hit by one of the two only (marching cubes interpolates edges linearly, the march blends
# trilinearly, so the two surfaces are close but not equal)
MARCH_MEDIAN, MARCH_P99, MARCH_ONLY_ONE = 0.02, 0.2, 0.005


def test_raster_depth_against_the_march_of_the_same_sdf():
    import mesh_ref
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("tiny")
    _, H_, W_ = s["depth"].shape
    vs = float(s["voxel_size"])
    rts, cam = rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"])
    m = mesh_ref.extract(s["xyz"], s["sdf0"], s["weight"], s["rgb"], vs, False)
    g = rr.Grid(s["xyz"], s["sdf0"], s["albedo"], s["weight"], vs)
    for f in (0, 3):
        v = rr.render_view(g, rts[f], cam, W_, H_, photometric=False)
        r = ra.rasterize(m, rts[f:f + 1], cam, W_, H_)
        hit_r = r["face"][0] >= 0
        both = v["hit"] & hit_r
        d = np.abs(v["depth"][both].astype(np.float64) - r["depth"][0][both]) / vs
        print(f, int(both.sum()), np.median(d), np.percentile(d, 99))
        assert both.sum() > 5000
        assert np.median(d) <= MARCH_MEDIAN and np.percentile(d, 99) <= MARCH_P99
        assert (v["hit"] ^ hit_r).sum() <= MARCH_ONLY_ONE * both.sum()


# Measured (restatement, tiny, vertex colours recomputed and the texture baked from the even keyframes, 12 texels per face, K = 5):
# mean |rendered - frame| over the covered pixels of the odd keyframes, averaged over R, G, B: full mesh 21.99 (texture) / 23.62
# (vertex colours), simplified at 4 voxels 22.90 / 29.38.  Small gives 21.10 / 24.03 and 23.26 / 35.35 (not run here: 35 s).
HELD_OUT_BOUND = {None: 22.8, 4: 26.0}


@pytest.mark.parametrize("cell", [None, 4])
def test_texture_beats_vertex_colours_on_held_out_keyframes(cell):
    import mesh_ref
    import mesh_simplify_ref as msr
    import oracle
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = config_scene("tiny")
    col = make_color_frames(s)
    F = len(s["poses"])
    even, odd = np.arange(0, F, 2), np.arange(1, F, 2)
    se = dict(s, lum=s["lum"][even], depth=s["depth"][even], poses=s["poses"][even])
    o = oracle.Oracle(threads=4)
    o.load_scene(se)
    o.set_color_frames(col[even])
    o.recompute_colors(0.02, 5)
    vs = float(s["voxel_size"])
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], o.colors(), vs, False)
    if cell:
        m = msr.simplify(m, cell * vs)
    rts, cam = rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"])
    _, H_, W_ = s["depth"].shape
    b = tr.bake(m, s["depth"][even], col[even], rts[even], cam, 12, 0.02, 5)
    err = {}
    for c in ("texture", "vertex"):
        r = ra.rasterize(m, rts, cam, W_, H_, color=c, texture=(b["image"], 12), depth=s["depth"], bgr=col, ids=list(odd))
        n = sum(st["color_count"] for st in r["stats"])
        err[c] = sum(sum(st["color_abs"]) for st in r["stats"]) / (3 * n)
    print(cell, err)
    assert err["texture"] <= HELD_OUT_BOUND[cell] < err["vertex"]
