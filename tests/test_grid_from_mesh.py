"""The numpy restatement of the voxel grid from a mesh (tests/grid_from_mesh_ref.py) against geometry with a known signed distance, and
mesh.load_ply.  No GPU: tests/test_gpu_zz_grid_from_mesh.py holds the device to the restatement byte for byte."""
import os

import numpy as np
import pytest

import distance_ref as dr
import grid_from_mesh_ref as gr

HERE = os.path.dirname(os.path.abspath(__file__))
VS = 0.01


def _rotation(w):
    from intrinsic3d_b200.scene import aa_to_rotation
    return aa_to_rotation(np.asarray(w, np.float64))


def _check_exact(out, sdf_true, tol):
    """|sdf| equals the exact distance to float accuracy and every sign away from the surface is right"""
    p = out["xyz"].astype(np.float64) * np.float64(np.float32(VS))
    t = sdf_true(p)
    np.testing.assert_allclose(np.abs(out["sdf"]), np.abs(t), rtol=0, atol=tol)
    far = np.abs(t) > tol
    assert (np.sign(out["sdf"][far]) == np.sign(t[far])).all()
    return t


BOXES = {
    "aligned": (np.array([-0.043, -0.031, -0.0275]), np.array([0.041, 0.052, 0.0385]), np.eye(3), np.zeros(3)),
    "rotated": (np.array([-0.04, -0.03, -0.035]), np.array([0.045, 0.05, 0.03]), _rotation([0.3, -0.5, 0.8]), np.array([0.0013, -0.0021, 0.0007])),
}


@pytest.mark.parametrize("name", sorted(BOXES))
def test_box_sign_and_distance(name):
    lo, hi, R, t = BOXES[name]
    mesh = gr.box_mesh(lo, hi, R, t)
    out = gr.grid_from_mesh(mesh, VS, 3.0)
    truth = _check_exact(out, lambda p: gr.box_sdf(p, lo, hi, R, t), 2e-8)
    assert out["num_boundary_edges"] == 0 and out["num_dropped_rim"] == 0
    assert (out["sdf"] < 0).any() and (out["sdf"] > 0).any()
    assert len(np.unique(out["feature"])) >= 4           # vertices, edges and interiors are all closest features


PRISMS = {
    "l": lambda: gr.l_prism(0.04, np.array([-0.0312, -0.0287, -0.0193])),
    "wedge": lambda: gr.wedge(0.08, 25.0, 0.05, np.array([-0.0412, -0.0037, -0.0231])),
}


@pytest.mark.parametrize("name", sorted(PRISMS))
def test_prism_concave_and_sharp_features(name):
    mesh, sdf = PRISMS[name]()
    out = gr.grid_from_mesh(mesh, VS, 3.0)
    truth = _check_exact(out, sdf, 2e-8)
    assert out["num_boundary_edges"] == 0 and (out["sdf"] < 0).any()
    if name == "wedge":
        # the nearest face's own normal signs some voxels by the knife edge wrongly: the sign test above can fail
        fs = gr.face_normal_signs(mesh, out, VS)
        far = np.abs(truth) > 2e-8
        assert (fs[far] != np.sign(truth[far])).any()


def test_welding_gives_the_same_grid():
    lo, hi, R, t = BOXES["rotated"]
    mesh = gr.box_mesh(lo, hi, R, t)
    a, b = gr.grid_from_mesh(mesh, VS, 3.0), gr.grid_from_mesh(gr.split_vertices(mesh), VS, 3.0)
    for k in ("xyz", "sdf", "face", "feature"):
        assert a[k].tobytes() == b[k].tobytes(), k
    assert b["num_welded"] == 8


def test_open_patch():
    z = 0.00337
    mesh = gr.square_patch(-0.0405, 0.0395, z, 3)
    out = gr.grid_from_mesh(mesh, VS, 3.0)
    p = out["xyz"].astype(np.float64) * np.float64(np.float32(VS))
    inner = (np.abs(p[:, 0] + 0.0005) < 0.04) & (np.abs(p[:, 1] + 0.0005) < 0.04)
    assert (np.sign(out["sdf"][inner]) == np.sign(p[inner, 2] - z)).all()
    np.testing.assert_allclose(np.abs(out["sdf"][inner]), np.abs(p[inner, 2] - z), rtol=0, atol=1e-8)
    # beyond the rim nothing, over it the 60 degree rule: kept iff |z - z0| >= |p - q| / 2, q the nearest point of the square
    q = np.clip(p[:, :2], -0.0405, 0.0395)
    d = np.linalg.norm(np.c_[p[:, :2] - q, p[:, 2] - z], axis=1)
    assert (d <= 3 * VS + 1e-7).all()
    assert (np.abs(p[~inner, 2] - z) >= 0.5 * d[~inner] - 1e-9).all()
    assert out["num_dropped_rim"] > 0 and out["num_boundary_edges"] == 12
    # every lattice point over the rim within the band that the rule keeps is there
    c = gr.candidates(mesh, VS, 3.0)
    pc = c.astype(np.float64) * np.float64(np.float32(VS))
    qc = np.clip(pc[:, :2], -0.0405, 0.0395)
    dc = np.linalg.norm(np.c_[pc[:, :2] - qc, pc[:, 2] - z], axis=1)
    want = (dc <= 3 * VS - 1e-7) & (np.abs(pc[:, 2] - z) >= 0.5 * dc + 1e-7)
    have = set(map(tuple, out["xyz"].tolist()))
    assert all(tuple(x) in have for x in c[want].tolist())


def _truth_checks(name, n_theta):
    import torch
    from intrinsic3d_b200.scene import _implicit, _truth_geometry, config_geometry, config_scene, truth_mesh, truth_mesh_error
    geo = config_geometry(name)
    mesh = truth_mesh(n_theta, **geo)
    err = truth_mesh_error(mesh, **geo)
    rho0, centre, bump, vs = _truth_geometry(**geo)
    out = gr.grid_from_mesh(mesh, vs, 3.0)
    c = torch.tensor(centre, dtype=torch.float64)
    p = torch.from_numpy(out["xyz"].astype(np.float64) * vs)
    f = _implicit(p, c, rho0, bump).numpy()
    # L: the largest gradient magnitude of the implicit over the band, by central differences
    h = 1e-6
    g = np.stack([(_implicit(p + h * torch.eye(3, dtype=torch.float64)[k], c, rho0, bump) - _implicit(p - h * torch.eye(3, dtype=torch.float64)[k], c,
                                                                                                      rho0, bump)).numpy() / (2 * h) for k in range(3)], 1)
    L = np.linalg.norm(g, axis=1).max()
    eps = 1e-6 * vs
    s = out["sdf"]
    sure = np.abs(f) > err + eps
    assert (np.sign(s[sure]) == np.sign(f[sure])).all()
    assert (np.abs(s) <= np.abs(f) + err + eps).all()
    assert (np.abs(s) >= np.abs(f) / L - err - eps).all()
    assert out["num_boundary_edges"] == 0 and out["num_dropped_rim"] == 0
    # the emitted set is make_scene's except within the radial-versus-Euclidean slack of the band edge
    sc = config_scene(name)
    b = float(np.float32(3.0) * np.float32(vs))
    mine, theirs = set(map(tuple, out["xyz"].tolist())), set(map(tuple, sc["xyz"].tolist()))
    for x in mine ^ theirs:
        fx = float(_implicit(torch.tensor(x, dtype=torch.float64) * vs, c, rho0, bump))
        assert b - err - eps < abs(fx) <= L * (b + err) + eps, (x, fx)
    return out, L


def test_truth_mesh_tiny():
    out, L = _truth_checks("tiny", 128)
    assert 1.0 < L < 2.0


def test_golden_fixture():
    g = np.load(os.path.join(HERE, "golden", "tiny_grid_from_mesh.npz"))
    mesh = dict(vertices=g["vertices"], faces=g["faces"])
    out = gr.grid_from_mesh(mesh, float(g["voxel_size"]), float(g["band"]))
    for k in ("xyz", "sdf", "face", "feature"):
        assert out[k].tobytes() == g[k].tobytes(), k


def test_point_tri_feature_keeps_the_distance():
    rng = np.random.default_rng(3)
    P = rng.normal(size=(4000, 3)).astype(np.float32)
    a, b, c = (rng.normal(size=(4000, 3)).astype(np.float32) for _ in range(3))
    c[:500] = a[:500] + np.float32(0.5) * (b[:500] - a[:500])         # degenerate (collinear) faces: the edge fallback
    c[500:600] = a[500:600] + np.float32(1e-4) * rng.normal(size=(100, 3)).astype(np.float32) + (b[500:600] - a[500:600])   # slivers
    d2 = dr.point_tri_d2(P, a, b, c)
    d2f, feat, dv = gr.point_tri_feature(P, a, b, c)
    assert d2.tobytes() == d2f.tobytes()
    np.testing.assert_allclose(dr._dot(dv, dv), d2, rtol=1e-6, atol=0)
    assert set(np.unique(feat)) == set(range(7))


# ---- load_ply -----------------------------------------------------------------------------------------------------------------------
def _mesh():
    lo, hi, R, t = BOXES["rotated"]
    m = gr.box_mesh(lo, hi, R, t)
    m["colors"] = np.arange(24, dtype=np.uint8).reshape(8, 3)
    return m


def test_load_ply_round_trips_save_ply(tmp_path):
    from intrinsic3d_b200 import mesh as M
    m = _mesh()
    path = tmp_path / "a.ply"
    M.save_ply(path, m)
    r = M.load_ply(path)
    for k in ("vertices", "colors", "faces"):
        assert r[k].dtype == m[k].dtype and r[k].tobytes() == m[k].tobytes(), k


def test_load_ply_ascii_and_double(tmp_path):
    from intrinsic3d_b200 import mesh as M
    m = _mesh()
    v, f = m["vertices"], m["faces"]
    hdr = ["ply", "format ascii 1.0", "comment test", f"element vertex {len(v)}", "property float x", "property float y", "property float z",
           "property float nx", f"element face {len(f)}", "property list uchar int vertex_index", "property uchar flags", "end_header"]
    lines = ["%.9g %.9g %.9g 0.5" % tuple(map(float, p)) for p in v] + ["3 %d %d %d 7" % tuple(x) for x in f]
    (tmp_path / "b.ply").write_text("\n".join(hdr + lines) + "\n")
    r = M.load_ply(tmp_path / "b.ply")
    assert r["vertices"].tobytes() == v.tobytes() and r["faces"].tobytes() == f.tobytes() and not r["colors"].any()
    # binary with double coordinates and an extra element
    hdr = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty double x\nproperty double y\nproperty double z\nproperty uchar q\n"
           "element face %d\nproperty list uchar uint vertex_indices\nelement junk 2\nproperty int a\nend_header\n" % (len(v), len(f))).encode()
    vr = np.empty(len(v), np.dtype([("p", "<f8", 3), ("q", "u1")]))
    vr["p"], vr["q"] = v.astype(np.float64), 9
    fr = np.empty(len(f), np.dtype([("n", "u1"), ("i", "<u4", 3)]))
    fr["n"], fr["i"] = 3, f
    (tmp_path / "c.ply").write_bytes(hdr + vr.tobytes() + fr.tobytes() + np.arange(2, dtype="<i4").tobytes())
    r = M.load_ply(tmp_path / "c.ply")
    assert r["vertices"].tobytes() == v.tobytes() and r["faces"].tobytes() == f.tobytes()


def test_load_ply_refuses_polygons(tmp_path):
    from intrinsic3d_b200 import mesh as M
    txt = "ply\nformat ascii 1.0\nelement vertex 4\nproperty float x\nproperty float y\nproperty float z\nelement face 1\n" \
          "property list uchar int vertex_indices\nend_header\n0 0 0\n1 0 0\n1 1 0\n0 1 0\n4 0 1 2 3\n"
    (tmp_path / "q.ply").write_text(txt)
    with pytest.raises(ValueError, match="not a triangle"):
        M.load_ply(tmp_path / "q.ply")
    hdr = b"ply\nformat binary_little_endian 1.0\nelement vertex 4\nproperty float x\nproperty float y\nproperty float z\nelement face 2\n" \
          b"property list uchar int vertex_indices\nend_header\n"
    body = np.zeros(12, "<f4").tobytes() + bytes([3]) + np.array([0, 1, 2], "<i4").tobytes() + bytes([4]) + np.array([0, 1, 2, 3], "<i4").tobytes()
    (tmp_path / "q2.ply").write_bytes(hdr + body)
    with pytest.raises(ValueError, match="not a triangle"):
        M.load_ply(tmp_path / "q2.ply")
