"""GPU tests of the rasterizer (i3d_rasterize_keyframes, i3d_rasterize_views, i3d_download_raster) against the numpy restatement
tests/raster_ref.py.  Explicitly rounded float arithmetic, 64-bit integer atomics and fixed-order double sums: the bar is BYTE-EQUAL
planes and integer statistics, depth sums to 1e-12."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
PLANES = ("depth", "face", "bary", "normal", "rgb")
DIST = np.array([0.03, -0.01, 0.004, 0.002, -0.0015])


def _engine(s, col):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(s)
    e.upload_color_frames(col)
    return e


def _scene(name, distort=False, device=None):
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = dict(config_scene(name, device=device) if device else config_scene(name))
    if distort:
        s["dist"] = DIST
    return s, make_color_frames(s)


def _cam(e):
    import render_ref as rr
    st = e.download_state()
    return rr.pose_rt(st["poses"]), rr.camera(st["intr"], st["dist"])


def _same_stats(g, r):
    for a, b in zip(g, r):
        for k in ("num_covered", "num_observed", "depth_count", "color_count", "color_abs", "color_sq"):
            assert a[k] == b[k], (k, a[k], b[k])
        for k in ("depth_abs", "depth_sq"):
            assert abs(a[k] - b[k]) <= 1e-12 * max(1.0, abs(b[k])), (k, a[k], b[k])


def _check_keyframes(e, s, col, mesh, ids, color="vertex", texture=None):
    import raster_ref as ra
    rt, cam = _cam(e)
    _, H, W = s["depth"].shape
    g = e.rasterize_keyframes(ids, color)
    r = ra.rasterize(mesh, rt, cam, W, H, color=color, texture=texture, depth=s["depth"], bgr=col, ids=list(ids))
    for k in PLANES:
        assert g[k].tobytes() == r[k].tobytes(), k
    _same_stats(g["stats"], r["stats"])
    i = g["info"]
    assert i.num_tests > 0 and i.num_covered == sum(st["num_covered"] for st in r["stats"]) and i.ms_faces > 0
    return g


def test_tiny_meshes_colours_and_binning(tiny_scene):
    s = tiny_scene
    from intrinsic3d_b200.scene import make_color_frames
    col = make_color_frames(s)
    e = _engine(s, col)
    vs = float(s["voxel_size"])
    ids = list(range(e.F))
    for src in ("fused", "refined"):
        m = e.extract_mesh(src, True)
        _check_keyframes(e, s, col, m, ids)
    for cell in (2, 4):
        e.extract_mesh("refined", False)
        m = e.simplify_mesh(cell * vs)
        g = _check_keyframes(e, s, col, m, ids)
        b = e.bake_texture(8)
        t = _check_keyframes(e, s, col, m, ids, "texture", (b["image"], 8))
        assert t["rgb"].tobytes() != g["rgb"].tobytes()
        e.set_raster_binning(False)
        for color in ("vertex", "texture"):
            off = e.rasterize_keyframes(ids, color)
            ref = g if color == "vertex" else t
            assert all(off[k].tobytes() == ref[k].tobytes() for k in PLANES) and off["stats"] == ref["stats"]
            assert off["info"].num_tests > ref["info"].num_tests
        e.set_raster_binning(True)
    st = e.rasterize_keyframes(ids, None, planes=())
    assert set(st) == {"stats", "info"} and all(x["color_count"] == 0 for x in st["stats"])


def test_small_distortion_and_binning_off():
    s, col = _scene("small", distort=True)
    e = _engine(s, col)
    m = e.extract_mesh("refined", True)
    ids = list(range(e.F))
    g = _check_keyframes(e, s, col, m, ids)
    b = e.bake_texture(12)
    _check_keyframes(e, s, col, m, [1, 4, 6], "texture", (b["image"], 12))
    e.set_raster_binning(False)
    off = e.rasterize_keyframes(ids, "vertex")
    assert all(off[k].tobytes() == g[k].tobytes() for k in PLANES) and off["stats"] == g["stats"]


def test_views_odd_sizes_and_inside_the_box(tiny_scene):
    import raster_ref as ra
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    e = _engine(s, col)
    m = e.extract_mesh("refined", True)
    b = e.bake_texture(8)
    rt, _ = _cam(e)
    V = m["vertices"]
    c = (V.min(0) + V.max(0)) / 2
    inside = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, -c[0], -c[1], -c[2]], np.float32)        # camera at the box centre
    poses = np.stack([rt[0], rt[3], inside]).astype(np.float32)
    for W, H, d in ((37, 29, np.zeros(5)), (123, 77, DIST)):
        cam = dict(fx=0.9 * W, fy=0.9 * W, cx=(W - 1) / 2 + 0.3, cy=(H - 1) / 2 - 0.2, width=W, height=H, distortion=d)
        rc = dict(fx=np.float32(cam["fx"]), fy=np.float32(cam["fy"]), cx=np.float32(cam["cx"]), cy=np.float32(cam["cy"]), d=d.astype(np.float32))
        for color, tex in (("vertex", None), ("texture", (b["image"], 8))):
            g = e.rasterize_views(cam, poses, color)
            r = ra.rasterize(m, poses, rc, W, H, color=color, texture=tex)
            for k in PLANES:
                assert g[k].tobytes() == r[k].tobytes(), (W, k)
            assert g["info"].num_straddling > 0 and (g["face"][2] >= 0).any()
        e.set_raster_binning(False)
        off = e.rasterize_views(cam, poses, "vertex")
        e.set_raster_binning(True)
        assert all(off[k].tobytes() == ra.rasterize(m, poses, rc, W, H, color="vertex")[k].tobytes() for k in PLANES)


def test_c2_subset_and_batch_independence():
    import torch
    s, col = _scene("c2", device="cuda" if torch.cuda.is_available() else "cpu")
    e = _engine(s, col)
    m = e.extract_mesh("refined", False)
    _check_keyframes(e, s, col, m, [0, 17, 33])
    m4 = e.simplify_mesh(4 * float(s["voxel_size"]))
    _check_keyframes(e, s, col, m4, [5, 40])
    # a view's bytes do not depend on the batch it is in
    one = e.rasterize_keyframes([7], "vertex")
    many = e.rasterize_keyframes([3, 7, 9], "vertex")
    assert all(one[k][0].tobytes() == many[k][1].tobytes() for k in PLANES) and one["stats"][0] == many["stats"][1]
    # binning off on a small view
    cam = dict(fx=60.0, fy=60.0, cx=31.5, cy=23.5, width=64, height=48)
    rt, _ = _cam(e)
    g = e.rasterize_views(cam, rt[:1])
    e.set_raster_binning(False)
    off = e.rasterize_views(cam, rt[:1])
    assert all(off[k].tobytes() == g[k].tobytes() for k in PLANES) and (g["face"] >= 0).any()


def test_c3_run_to_run_and_engine_to_engine():
    import torch
    s, col = _scene("c3", device="cuda" if torch.cuda.is_available() else "cpu")
    engines = [_engine(s, col), _engine(s, col)]
    ids = list(range(engines[0].F))
    res = []
    for e in (engines[0], engines[0], engines[1]):
        if e is not engines[0] or not res:
            e.extract_mesh("refined", False)
        st = e.rasterize_keyframes(ids, "vertex", planes=())
        pl = e.rasterize_keyframes([0, 99, 199], "vertex")
        res.append((st["stats"], pl))
    for st, pl in res[1:]:
        assert st == res[0][0]
        assert all(pl[k].tobytes() == res[0][1][k].tobytes() for k in PLANES)
    print("c3", res[0][1]["info"].as_dict())
    for e in engines:
        e.close()


def test_golden_fixture(tiny_scene):
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    z = np.load(os.path.join(HERE, "golden", "tiny_raster.npz"))
    e = _engine(s, make_color_frames(s))
    m = e.extract_mesh("refined", True)
    assert m["faces"].tobytes() == z["faces"].tobytes()
    g = e.rasterize_keyframes(z["ids"], "vertex")
    for k in PLANES:
        assert g[k].tobytes() == z[k].tobytes(), k
    got = np.array([[st["num_covered"], st["num_observed"], st["depth_count"], st["color_count"], *st["color_abs"], *st["color_sq"]]
                    for st in g["stats"]], np.int64)
    assert got.tobytes() == z["counts"].tobytes()
    assert np.allclose([[st["depth_abs"], st["depth_sq"]] for st in g["stats"]], z["sums"], rtol=1e-12, atol=0)


def test_refusals_leave_the_planes_and_lifetime(tiny_scene):
    import ctypes as C
    from intrinsic3d_b200.ctypes_defs import I3DRasterCamera, I3DRasterInfo, I3DRasterParams, I3DRasterStats
    from intrinsic3d_b200.engine import Engine, _p
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    e0 = Engine(0)
    with pytest.raises(RuntimeError, match="no mesh"):
        e0.rasterize_keyframes([0])
    e0.close()
    e = Engine(0)
    e.load_scene(s)
    e.extract_mesh("refined", True)
    with pytest.raises(RuntimeError, match="colour frames"):
        e.rasterize_keyframes([0], "vertex")
    e.upload_color_frames(col)
    with pytest.raises(RuntimeError, match="texture"):
        e.rasterize_keyframes([0], "texture")
    ref = e.rasterize_keyframes([0, 1], "vertex")
    L, h = e.L, e.h
    ids = np.array([0], np.int32)
    good = I3DRasterParams(31, 1)
    cam = I3DRasterCamera(100.0, 100.0, 20.0, 15.0, (C.c_float * 5)(), 40, 30)
    pose = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 1], np.float32)
    st, info = (I3DRasterStats * 2)(), I3DRasterInfo()
    bad_calls = [
        lambda: L.i3d_rasterize_keyframes(h, 0, _p(ids, C.c_int32), C.byref(good), st, C.byref(info)),
        lambda: L.i3d_rasterize_keyframes(h, 1, _p(np.array([e.F], np.int32), C.c_int32), C.byref(good), st, C.byref(info)),
        lambda: L.i3d_rasterize_keyframes(h, 1, _p(np.array([-1], np.int32), C.c_int32), C.byref(good), st, C.byref(info)),
        lambda: L.i3d_rasterize_keyframes(h, 1, None, C.byref(good), st, C.byref(info)),
        lambda: L.i3d_rasterize_keyframes(h, 1, _p(ids, C.c_int32), C.byref(I3DRasterParams(32, 1)), st, C.byref(info)),
        lambda: L.i3d_rasterize_keyframes(h, 1, _p(ids, C.c_int32), C.byref(I3DRasterParams(-1, 1)), st, C.byref(info)),
        lambda: L.i3d_rasterize_keyframes(h, 1, _p(ids, C.c_int32), C.byref(I3DRasterParams(31, 3)), st, C.byref(info)),
        lambda: L.i3d_rasterize_keyframes(h, 1, _p(ids, C.c_int32), None, st, C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, None, _p(pose, C.c_float), C.byref(good), C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, C.byref(cam), None, C.byref(good), C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, C.byref(cam), _p(np.full(12, np.nan, np.float32), C.c_float), C.byref(good), C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, C.byref(I3DRasterCamera(100.0, 100.0, 20.0, 15.0, (C.c_float * 5)(), 0, 30)), _p(pose, C.c_float),
                                      C.byref(good), C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, C.byref(I3DRasterCamera(100.0, 100.0, 20.0, 15.0, (C.c_float * 5)(), 8193, 30)), _p(pose, C.c_float),
                                      C.byref(good), C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, C.byref(I3DRasterCamera(-1.0, 100.0, 20.0, 15.0, (C.c_float * 5)(), 40, 30)), _p(pose, C.c_float),
                                      C.byref(good), C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, C.byref(I3DRasterCamera(100.0, 100.0, float("nan"), 15.0, (C.c_float * 5)(), 40, 30)),
                                      _p(pose, C.c_float), C.byref(good), C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, C.byref(I3DRasterCamera(100.0, 100.0, 20.0, 15.0, (C.c_float * 5)(float("inf")), 40, 30)),
                                      _p(pose, C.c_float), C.byref(good), C.byref(info)),
        lambda: L.i3d_rasterize_views(h, 1, C.byref(cam), _p(pose, C.c_float), C.byref(I3DRasterParams(31, 2)), C.byref(info)),
    ]
    for k, call in enumerate(bad_calls):
        assert call() != 0, k
        assert L.i3d_last_error(h).decode(), k
        d = np.empty((2,) + ref["depth"].shape[1:], np.float32)
        assert L.i3d_download_raster(h, _p(d, C.c_float), None, None, None, None) == 0
        assert d.tobytes() == ref["depth"].tobytes(), k
    # a plane that was not rendered
    e.rasterize_keyframes([0], "vertex", planes=("depth",))
    f = np.empty(ref["face"][:1].shape, np.int32)
    assert L.i3d_download_raster(h, None, _p(f, C.c_int32), None, None, None) != 0
    # lifetime: extraction, simplification, pruning and a frame change drop the planes; a camera change does not
    d = np.empty(ref["depth"][:1].shape, np.float32)

    def have():
        return L.i3d_download_raster(h, _p(d, C.c_float), None, None, None, None) == 0
    e.set_camera(s["poses"] * 1.0001, s["intr"], s["dist"])
    assert have()
    e.extract_mesh("refined", True)
    assert not have()
    e.rasterize_keyframes([0], "vertex")
    e.simplify_mesh(4 * float(s["voxel_size"]))
    assert not have()
    with pytest.raises(RuntimeError, match="texture"):             # the texture went with the simplification
        e.rasterize_keyframes([0], "texture")
    e.rasterize_keyframes([0], "vertex")
    e.upload_frames(s["lum"], s["depth"])
    assert not have()
    e.rasterize_views(dict(fx=50.0, fy=50.0, cx=20.0, cy=15.0, width=40, height=30), pose[None])
    e.upload_frames(s["lum"], s["depth"])
    assert have()                                                  # a frame change keeps the planes of new views
    e.clear_voxels_outside_thin_shell(float(s["thres_shell"]))
    assert not have()
    e.close()


def test_no_side_effects(tiny_scene):
    """a GN iteration, a recolouring, a render, a bake, a distance call and the next extraction give the same bytes with and without
    raster calls in between"""
    from intrinsic3d_b200.ctypes_defs import default_params
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    out = []
    for with_raster in (False, True):
        e = _engine(s, col)
        r = {}

        def raster():
            if with_raster:
                e.rasterize_keyframes(list(range(e.F)), "vertex")
                e.rasterize_views(dict(fx=50.0, fy=50.0, cx=20.0, cy=15.0, width=40, height=30), np.eye(3, 4, dtype=np.float32).reshape(1, 12))
        m = e.extract_mesh("refined", True)
        e.upload_reference_mesh(m)
        raster()
        p = default_params()
        p.thres_shell = s["thres_shell"]
        p.forced_cg_iterations = 4
        e.gn_iteration(p)
        st = e.download_state()
        r["gn"] = b"".join(np.ascontiguousarray(st[k]).tobytes() for k in sorted(st) if isinstance(st[k], np.ndarray))
        raster()
        e.recompute_colors(0.02, 5)
        r["colors"] = e.download_colors().tobytes()
        raster()
        r["render"] = e.render_keyframes([0, 1], planes=("depth", "normal"), photometric=False)["depth"].tobytes()
        m = e.extract_mesh("refined", True)
        raster()
        r["bake"] = e.bake_texture(8)["image"].tobytes()
        raster()
        r["dist"] = e.surface_distance()["vertex_distance"].tobytes()
        raster()
        m = e.extract_mesh("refined", True)
        r["mesh"] = m["vertices"].tobytes() + m["faces"].tobytes() + m["colors"].tobytes()
        out.append(r)
        e.close()
    for k in out[0]:
        assert out[0][k] == out[1][k], k


def test_passes_of_few_views_give_the_same_bytes(tiny_scene):
    """a call split into passes (views v0 > 0 of a pass: their keys, partials and sums) gives the bytes of one pass"""
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    e = _engine(s, make_color_frames(s))
    e.extract_mesh("refined", True)
    ids = list(range(e.F))
    one = e.rasterize_keyframes(ids, "vertex")
    cam = dict(fx=40.0, fy=40.0, cx=20.0, cy=14.5, width=41, height=30, distortion=DIST)
    rt, _ = _cam(e)
    vone = e.rasterize_views(cam, rt)
    for views in (1, 4):
        e.set_raster_batch(views)
        split = e.rasterize_keyframes(ids, "vertex")
        assert all(split[k].tobytes() == one[k].tobytes() for k in PLANES) and split["stats"] == one["stats"], views
        vs = e.rasterize_views(cam, rt)
        assert all(vs[k].tobytes() == vone[k].tobytes() for k in PLANES), views
    e.set_raster_batch(0)
    with pytest.raises(RuntimeError):
        e.set_raster_batch(-1)
    e.close()
