"""GPU tests of the surface distance (i3d_upload_reference_mesh, i3d_surface_distance, i3d_download_surface_distance) against the numpy
restatement tests/distance_ref.py.  Explicitly rounded float arithmetic and a fixed summation order: the bar is BYTE-EQUAL per-sample and
per-vertex (d^2, face), equal counts, and statistics within 1e-12 of the float64 restatement."""
import ctypes as C
import os

import numpy as np
import pytest

import distance_ref as dr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
STATS = ("area", "unmatched_area", "mean", "rms", "max")


def _engine(s):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(s)
    e.debug_set_keep_distance_samples(True)
    return e


def _truth(name, n_theta=None):
    from intrinsic3d_b200.scene import config_geometry, truth_mesh
    return truth_mesh(n_theta, **config_geometry(name))


def _device(e, L, maxd, taus, cell=None):
    g = e.surface_distance(taus, maxd, L, cell)
    for d, side in enumerate(("accuracy", "completeness")):
        g[side + "_d2"], g[side + "_face"] = e.debug_distance_samples(d, g[side]["num_samples"])
    return g


def _check(e, mesh_a, mesh_b, L, maxd, taus, cell=None):
    """the resident mesh (mesh_a as downloaded) against the uploaded reference mesh_b, on the engine and in the restatement"""
    g = _device(e, L, maxd, taus, cell)
    r = dr.distance(mesh_a, mesh_b, L, maxd, taus)
    for side in ("accuracy", "completeness"):
        assert g[side + "_d2"].tobytes() == r[side + "_d2"].tobytes(), (side, L)
        assert g[side + "_face"].tobytes() == r[side + "_face"].tobytes(), (side, L)
        assert (g[side]["num_samples"], g[side]["num_matched"]) == (r[side]["num_samples"], r[side]["num_matched"])
        for k in STATS:
            np.testing.assert_allclose(g[side][k], r[side][k], rtol=1e-12, atol=0, err_msg=(side, k))
        np.testing.assert_allclose(g[side]["fraction"], r[side]["fraction"], rtol=1e-12, atol=0)
        assert g[side]["point_triangle_tests"] >= g[side]["num_matched"]
    for k in ("precision", "recall", "fscore"):
        np.testing.assert_allclose(g[k], r[k], rtol=1e-12, atol=0)
    assert g["vertex_distance"].tobytes() == r["vertex_distance"].tobytes() and g["vertex_face"].tobytes() == r["vertex_face"].tobytes()
    return g


def test_tiny_sources_meshes_and_references(tiny_scene):
    from intrinsic3d_b200.ctypes_defs import default_params
    s = tiny_scene
    vs = float(s["voxel_size"])
    taus = [0.1 * vs, 0.25 * vs, 0.5 * vs]
    e = _engine(s)
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    e.gn_iteration(p)
    truth = _truth("tiny", 64)
    e.upload_reference_mesh(truth)
    for src in ("fused", "refined"):
        m = e.extract_mesh(src, False)
        for L in (1, 2, 5):
            _check(e, m, truth, L, 2 * vs, taus)
    m = e.simplify_mesh(2 * vs)
    _check(e, m, truth, 2, 2 * vs, taus)
    # against another extraction, with a max_distance that leaves samples unmatched
    other = e.extract_mesh("fused", True)
    m = e.extract_mesh("refined", False)
    e.upload_reference_mesh(other)
    g = _check(e, m, other, 2, 0.05 * vs, [0.02 * vs])
    assert 0 < g["accuracy"]["num_matched"] < g["accuracy"]["num_samples"]


def test_small_scene(small_scene):
    s = small_scene
    vs = float(s["voxel_size"])
    e = _engine(s)
    truth = _truth("small")
    e.upload_reference_mesh(truth)
    m = e.extract_mesh("refined", False)
    _check(e, m, truth, 2, 2 * vs, [0.1 * vs, 0.5 * vs])
    _check(e, e.simplify_mesh(4 * vs), truth, 5, 2 * vs, [0.25 * vs])


def test_c2():
    import torch
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c2", device="cuda" if torch.cuda.is_available() else "cpu")
    vs = float(s["voxel_size"])
    e = _engine(s)
    truth = _truth("c2", 256)
    e.upload_reference_mesh(truth)
    m = e.extract_mesh("refined", False)
    g = _check(e, m, truth, 1, 2 * vs, [0.1 * vs, 0.25 * vs, 0.5 * vs])
    print("c2", len(m["faces"]), len(truth["faces"]), {k: g["info"].side[0].__getattribute__(k) for k in ("ms_grid", "ms_query", "ms_reduce")},
          g["fscore"])


def test_independent_of_the_grid(tiny_scene):
    s = tiny_scene
    vs = float(s["voxel_size"])
    e = _engine(s)
    e.upload_reference_mesh(_truth("tiny", 64))
    e.extract_mesh("refined", False)
    res = [_device(e, 2, 2 * vs, [0.25 * vs], cell) for cell in (None, 0.7 * vs, 5.0 * vs)]
    cells = [r["info"].side[0].cell_size for r in res]
    assert len(set(cells)) == 3, cells
    for r in res[1:]:
        for k in ("accuracy_d2", "accuracy_face", "completeness_d2", "completeness_face", "vertex_distance", "vertex_face"):
            assert r[k].tobytes() == res[0][k].tobytes(), k
        for side in ("accuracy", "completeness"):
            assert [r[side][k] for k in STATS] == [res[0][side][k] for k in STATS]
            assert r[side]["fraction"] == res[0][side]["fraction"]


def test_c3_two_calls_two_engines_bit_identical():
    import torch
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c3", device="cuda" if torch.cuda.is_available() else "cpu")
    vs = float(s["voxel_size"])
    truth = _truth("c3")
    out = []
    for e in (_engine(s), _engine(s)):
        e.extract_mesh("refined", False)
        e.upload_reference_mesh(truth)
        for _ in range(2):
            g = _device(e, 2, 2 * vs, [0.1 * vs, 0.25 * vs, 0.5 * vs])
            info = g["info"]
            stats = b"".join(bytes(info.side[d])[:type(info.side[d]).ms_grid.offset] for d in range(2))
            out.append((stats, bytes(info)[type(info).num_thresholds.offset:type(info).ms_vertices.offset],
                        b"".join(g[k].tobytes() for k in ("accuracy_d2", "accuracy_face", "completeness_d2", "completeness_face",
                                                          "vertex_distance", "vertex_face"))))
        print("c3", info.side[0].num_samples, info.side[1].num_samples, [(info.side[d].ms_grid, info.side[d].ms_query) for d in range(2)], g["fscore"])
        e.close()
    assert all(o == out[0] for o in out[1:])


def test_golden_fixture(tiny_scene):
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden_distance as mg
    g = np.load(os.path.join(HERE, "golden", "tiny_distance.npz"))
    e = _engine(tiny_scene)
    m = e.extract_mesh("refined", True)
    assert m["faces"].tobytes() == g["faces"].tobytes()
    e.upload_reference_mesh(mg.truth_mesh(mg.N_THETA, **mg.config_geometry("tiny")))
    r = _device(e, int(g["L"]), float(g["max_distance"]), [float(t) for t in g["thresholds"]])
    for k in ("accuracy_d2", "accuracy_face", "completeness_d2", "completeness_face", "vertex_distance", "vertex_face"):
        assert r[k].tobytes() == g[k].tobytes(), k
    for side in ("accuracy", "completeness"):
        np.testing.assert_allclose([r[side][k] for k in ("mean", "rms", "max", "area", "unmatched_area")] + r[side]["fraction"], g[side + "_stats"],
                                   rtol=1e-12, atol=0)


def _resident(e):
    from intrinsic3d_b200.engine import _p
    V, F = 100000, 200000
    out = dict(v=np.zeros((V, 3), np.float32), c=np.zeros((V, 3), np.uint8), f=np.zeros((F, 3), np.int32))
    assert e.L.i3d_download_mesh(e.h, _p(out["v"], C.c_float), _p(out["c"], C.c_uint8), _p(out["f"], C.c_int32)) == 0
    return b"".join(a.tobytes() for a in out.values())


def test_refusals_leave_state(tiny_scene):
    from intrinsic3d_b200.ctypes_defs import I3DDistanceInfo, I3DDistanceParams
    from intrinsic3d_b200.engine import _p, default_distance_params
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    vs = float(s["voxel_size"])
    info = I3DDistanceInfo()

    def call(e, L=2, maxd=2 * vs, cell=0.0, taus=(0.1 * vs, 0.5 * vs), nt=None):
        t = list(taus) + [0.0] * (8 - len(taus))
        prm = I3DDistanceParams(L, maxd, cell, len(taus) if nt is None else nt, (C.c_float * 8)(*t))
        return e.L.i3d_surface_distance(e.h, C.byref(prm), C.byref(info))

    def err(e):
        return e.L.i3d_last_error(e.h).decode()
    e = _engine(s)
    assert call(e) != 0 and "no mesh" in err(e)
    m = e.extract_mesh("refined", True)
    assert call(e) != 0 and "no reference" in err(e)
    assert e.L.i3d_download_surface_distance(e.h, None, None) != 0 and "no result" in err(e)
    truth = _truth("tiny", 32)
    e.upload_reference_mesh(truth)
    e.upload_color_frames(make_color_frames(s))
    tex = e.bake_texture(8)
    first = e.surface_distance([0.1 * vs], 2 * vs, 2)
    mesh0 = _resident(e)
    for args, msg in (((0,), "samples_per_edge"), ((17,), "samples_per_edge"), ((2, float("nan")), "max_distance"), ((2, 0.0), "max_distance"),
                      ((2, -1.0), "max_distance"), ((2, float("inf")), "max_distance"), ((2, 2 * vs, -1.0), "cell_size"),
                      ((2, 2 * vs, float("nan")), "cell_size"), ((2, 2 * vs, 0.0, (0.5 * vs, 0.1 * vs)), "thresholds"),
                      ((2, 2 * vs, 0.0, (float("nan"),)), "thresholds"), ((2, 2 * vs, 0.0, (3 * vs,)), "thresholds"),
                      ((2, 2 * vs, 0.0, (), -1), "num_thresholds"), ((2, 2 * vs, 0.0, (), 9), "num_thresholds"),
                      ((2, 2 * vs, 1e-5), "I3D_DISTANCE_MAX_CELLS")):
        assert call(e, *args) != 0, args
        assert msg in err(e), (args, err(e))
        assert _resident(e) == mesh0
        vd, vf = np.zeros(len(m["vertices"]), np.float32), np.zeros(len(m["vertices"]), np.int32)
        assert e.L.i3d_download_surface_distance(e.h, _p(vd, C.c_float), _p(vf, C.c_int32)) == 0
        assert vd.tobytes() == first["vertex_distance"].tobytes() and vf.tobytes() == first["vertex_face"].tobytes()
        img = np.zeros_like(tex["image"])
        assert e.L.i3d_download_texture(e.h, _p(img, C.c_uint8), None) == 0 and img.tobytes() == tex["image"].tobytes()
    assert e.L.i3d_surface_distance(e.h, None, C.byref(info)) != 0
    # reference uploads that are refused keep the previous reference
    v = np.ascontiguousarray(truth["vertices"])
    f = np.ascontiguousarray(truth["faces"])
    bad_f = f.copy()
    bad_f[3, 1] = len(v)
    neg_f = f.copy()
    neg_f[0, 0] = -1
    bad_v = v.copy()
    bad_v[5, 2] = np.inf
    for V, vp, F, fp, msg in ((0, v, len(f), f, "V > 0"), (len(v), v, 0, f, "F > 0"), (len(v), None, len(f), f, "NULL"), (len(v), v, len(f), None, "NULL"),
                              (len(v), v, len(f), bad_f, "outside"), (len(v), v, len(f), neg_f, "outside"), (len(v), bad_v, len(f), f, "not finite"),
                              (1 << 32, v, len(f), f, "int32")):
        assert e.L.i3d_upload_reference_mesh(e.h, V, _p(vp, C.c_float), F, _p(fp, C.c_int32)) != 0, msg
        assert msg in err(e), (msg, err(e))
    again = e.surface_distance([0.1 * vs], 2 * vs, 2)
    assert again["vertex_distance"].tobytes() == first["vertex_distance"].tobytes() and again["precision"] == first["precision"]
    # a mesh without faces
    import test_gpu_zz_mesh as tgm
    import test_mesh as tm
    xyz, sdf, w, rgb = tm.grid(tm._sphere((3.3, 2.6, 4.1), 2.2, half=4))
    e3 = tgm._engine_with(xyz, sdf, sdf, w, rgb, 0.004)
    e3.extract_mesh("refined")
    assert len(e3.simplify_mesh(1.0)["faces"]) == 0
    e3.upload_reference_mesh(truth)
    assert call(e3) != 0 and "no faces" in err(e3)
    # struct sizes and defaults
    p = default_distance_params()
    assert (p.samples_per_edge, p.num_thresholds, p.cell_size) == (2, 3, 0.0) and abs(p.max_distance - 0.01) < 1e-9
    assert e.L.i3d_sizeof_distance_params() == C.sizeof(I3DDistanceParams) == 48
    assert e.L.i3d_sizeof_distance_info() == C.sizeof(I3DDistanceInfo) == 592
    # the reference survives a change of the voxel set
    e.upsample_grid()
    e.extract_mesh("refined", False)
    assert e.surface_distance([0.1 * vs], 2 * vs, 1)["accuracy"]["num_samples"] > 0


def test_state_unchanged_by_distance(tiny_scene):
    """A GN iteration, a recolouring, a render, a bake and the next extraction are byte-identical with and without distance calls"""
    from intrinsic3d_b200.ctypes_defs import default_params
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    vs = float(s["voxel_size"])
    col = make_color_frames(s)
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    truth = _truth("tiny", 32)
    out = []
    for dist in (False, True):
        e = _engine(s)
        e.upload_color_frames(col)
        e.gn_iteration(p)
        e.extract_mesh("refined", True)
        if dist:
            e.upload_reference_mesh(truth)
            e.surface_distance([0.1 * vs], 2 * vs, 2)
            e.surface_distance([0.5 * vs], vs, 5, 3 * vs)
        info = e.gn_iteration(p)
        cnt = e.recompute_colors(0.02, 5)
        r = e.render_keyframes([0, 1])
        e.extract_mesh("refined", True)
        t = e.bake_texture(8)
        m = e.extract_mesh("fused", False)
        out.append((bytes(info)[:type(info).time_add.offset], e.download_state(), cnt, e.download_colors(), r, t, m))
    assert out[0][0] == out[1][0] and out[0][2] == out[1][2]
    for k in out[0][1]:
        assert out[0][1][k].tobytes() == out[1][1][k].tobytes(), k
    assert out[0][3].tobytes() == out[1][3].tobytes()
    for k in out[0][4]:
        if k != "stats":
            assert out[0][4][k].tobytes() == out[1][4][k].tobytes(), k
    assert out[0][5]["image"].tobytes() == out[1][5]["image"].tobytes() and out[0][5]["uv"].tobytes() == out[1][5]["uv"].tobytes()
    for k in ("vertices", "colors", "faces"):
        assert out[0][6][k].tobytes() == out[1][6][k].tobytes(), k
