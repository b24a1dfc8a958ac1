"""GPU tests of the keyframe renderer (i3d_render_keyframes / i3d_download_render) against the numpy restatement tests/render_ref.py on
the downloaded grid: planes byte-equal, counts exact, sums to 1e-12 relative.  Empty-space skipping on and off must give the same bytes."""
import ctypes as C
import os

import numpy as np
import pytest

import render_ref as rr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ALL = rr.PLANES
INTS = ("num_hit", "num_observed", "depth_count", "photo_count")
SUMS = ("depth_abs", "depth_sq", "photo_abs", "photo_sq")


def _same_stats(a, b, rel=1e-12):
    for k in INTS:
        assert a[k] == b[k], (k, a[k], b[k])
    for k in SUMS:
        assert abs(a[k] - b[k]) <= rel * max(abs(b[k]), 1e-300), (k, a[k], b[k])


def _bytes(out):
    return b"".join(out[p].tobytes() for p in ALL if p in out) + repr(out["stats"]).encode()


def _check(e, ids, source="refined", photometric=True, pyr_scale=1.0):
    """the engine's render of ids against the restatement of the downloaded grid, camera, SH and frames"""
    g = e.download_grid()
    st = e.download_state()
    sh, has = e.download_voxel_sh() if photometric else (None, None)
    lum, depth, _ = e.debug_frames()
    out = e.render_keyframes(ids, source, ALL if photometric else ("depth", "normal", "albedo"), photometric)
    ref = rr.render(rr.grid_of(g, source, sh, has), st["poses"], st["intr"], st["dist"], pyr_scale, list(ids), depth, lum, photometric)
    for p in out:
        if p != "stats":
            assert out[p].tobytes() == ref[p].tobytes(), (p, int((out[p] != ref[p]).sum()))
    for a, b in zip(out["stats"], ref["stats"]):
        _same_stats(a, b)
    return out, ref


def _skip_same(e, ids, source="refined", photometric=True):
    planes = ALL if photometric else ("depth", "normal", "albedo")
    e.set_render_skip(True)
    a = e.render_keyframes(ids, source, planes, photometric)
    na = e.phase_count("render_samples")
    e.set_render_skip(False)
    b = e.render_keyframes(ids, source, planes, photometric)
    nb = e.phase_count("render_samples")
    e.set_render_skip(True)
    assert _bytes(a) == _bytes(b)
    assert na <= nb
    return na, nb


def test_tiny_scene_bytes_equal(tiny_scene):
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    e = Engine(0)
    e.load_scene(s)
    for src in ("fused", "refined"):
        out, _ = _check(e, [0, 2, 5], src)
        assert all(st["num_hit"] > 1000 and st["photo_count"] > 500 for st in out["stats"]), out["stats"]
        print(src, e.phase_ms("render"), e.phase_count("render_samples"), _skip_same(e, [0, 2, 5], src))
    # lens distortion
    e.set_camera(s["poses"], s["intr"], np.array([0.1, -0.04, 0.01, 0.002, -0.003]))
    _check(e, [1, 4])
    _skip_same(e, [1, 4])
    # pyramid level 1: the same frame count at half the size, intrinsics * 0.5
    e.set_camera(s["poses"], s["intr"], s["dist"])
    e.upload_frames(s["lum"][:, ::2, ::2], s["depth"][:, ::2, ::2], 0.5)
    out, _ = _check(e, [0, 3], pyr_scale=0.5)
    assert out["depth"].shape == (2, 60, 80) and out["stats"][0]["num_hit"] > 200


def test_partial_sh_after_lighting_estimate(tiny_scene):
    """the per-voxel SH of the lighting estimate (only the thin shell has SH): renormalised over the corners that have it"""
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    e = Engine(0)
    e.load_scene(s)
    lp = engine.default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    lp.subvolume_size = 0.02
    e.estimate_lighting(lp)
    has = e.download_voxel_sh()[1]
    assert 0 < has.sum() < len(has)
    out, _ = _check(e, [0, 1, 2, 3, 4, 5])
    assert all(st["photo_count"] > 0 for st in out["stats"])


def test_golden_fixture_bytes_equal():
    from intrinsic3d_b200.engine import Engine
    g = np.load(os.path.join(HERE, "golden", "tiny_render.npz"))
    e = Engine(0)
    e.upload_grid(g["xyz"], g["sdf0"], g["sdf_refined"], g["albedo"], g["weight"], g["rgb"], float(g["voxel_size"]))
    e.upload_frames(g["lum"], g["depth"])
    e.set_camera(g["poses"], g["intr"], g["dist"])
    e.set_sh(g["sh"])
    out = e.render_keyframes([0, 1])
    for p in ALL:
        assert out[p].tobytes() == g["plane_" + p].tobytes(), p
    for i, st in enumerate(out["stats"]):
        assert [st[k] for k in INTS] == g["stats_int"][i].tolist()
        for j, k in enumerate(SUMS):
            assert abs(st[k] - g["stats_sum"][i, j]) <= 1e-12 * abs(g["stats_sum"][i, j])


def _constructed_engine(g, poses, W=33, H=27, f=30.0, dist=np.zeros(5), seed=3):
    from intrinsic3d_b200.engine import Engine
    rng = np.random.default_rng(seed)
    F = len(poses)
    depth = (0.2 + 0.2 * rng.random((F, H, W))).astype(np.float32)
    depth[rng.random((F, H, W)) < 0.1] = 0.0
    lum = rng.random((F, H, W)).astype(np.float32)
    e = Engine(0)
    e.upload_grid(g["xyz"], g["sdf0"], g["sdf_refined"], g["albedo"], g["weight"], g["rgb"], float(g["voxel_size"]))
    e.upload_frames(lum, depth)
    e.set_camera(np.asarray(poses, np.float64), np.array([f, f, (W - 1) / 2.0, (H - 1) / 2.0]), dist)
    e.set_sh(np.tile([0.7, 0.1, -0.2, 0.3, 0.02, -0.05, 0.04, 0.01, -0.03], (len(g["xyz"]), 1)))
    return e


def _sphere(centre_vox, radius_vox, vs, band=3.0):
    c = np.floor(np.asarray(centre_vox)).astype(int)
    r = int(np.ceil(radius_vox + band)) + 1
    ax = [np.arange(c[d] - r, c[d] + r + 1) for d in range(3)]
    X, Y, Z = np.meshgrid(*ax, indexing="ij")
    xyz = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)
    d = np.linalg.norm(xyz - np.asarray(centre_vox)[None, :], axis=1) - radius_vox
    keep = np.abs(d) <= band
    xyz, d = xyz[keep].astype(np.int32), d[keep] * float(np.float32(vs))
    n = len(xyz)
    return dict(xyz=xyz, sdf0=-d, sdf_refined=d, albedo=np.linspace(0.3, 0.9, n), weight=np.ones(n, np.float32),
                rgb=np.full((n, 3), 90, np.uint8), voxel_size=np.float32(vs))


def _check_constructed(e, ids, photometric=True):
    for src in ("fused", "refined"):
        out, _ = _check(e, ids, src, photometric)
        _skip_same(e, ids, src, photometric)
    return out


def test_constructed_grids_bytes_equal():
    import test_render as tr
    # a plane head-on and at an angle, seen from the origin
    for nrm in ((0, 0, 1), (0.3, -0.2, 1.0)):
        g = tr.plane_grid(nrm, 0.3)
        out = _check_constructed(_constructed_engine(g, [[0, 0, 0, 0, 0, 0], [0.05, 0.1, 0.0, 0.01, 0.0, 0.02]]), [0, 1])
        assert out["stats"][0]["num_hit"] > 500
    # missing corners (the hash probe of (1,1,1) and the neighbour table) and zero-weight corners
    g = tr.plane_grid((0.1, 0.2, 1.0), 0.3)
    rng = np.random.default_rng(8)
    keep = rng.random(len(g["xyz"])) > 0.04
    g = {k: (v[keep] if isinstance(v, np.ndarray) and v.ndim and len(v) == len(keep) else v) for k, v in g.items()}
    g["weight"][rng.random(len(g["xyz"])) < 0.04] = 0.0
    out = _check_constructed(_constructed_engine(g, [[0, 0, 0, 0, 0, 0]]), [0])
    assert 0 < out["stats"][0]["num_hit"] < 33 * 27
    # a sphere far from the origin (coordinates near 70000 voxels, voxel size 1), seen from 20 voxels in front of it
    c = np.array([70000.37, 70000.61, 70000.23])
    g = _sphere(c, 4.3, 1.0)
    out = _check_constructed(_constructed_engine(g, [[0, 0, 0, -c[0], -c[1], -(c[2] - 20.0)]], f=60.0), [0])
    assert out["stats"][0]["num_hit"] > 50
    # a sphere of radius 6 voxels: the camera inside the voxel box but outside the surface; the camera at the centre (every ray starts
    # inside the surface: no crossing from > 0 to <= 0, so no hit); a camera looking away (no hit)
    g = _sphere((0.0, 0.0, 0.0), 6.0, 0.01)
    e = _constructed_engine(g, [[0, 0, 0, 0, 0, 0.08], [0, 0, 0, 0, 0, 0], [0, np.pi, 0, 0, 0, -0.3]], f=20.0)
    out = _check_constructed(e, [0, 1, 2])
    assert out["stats"][0]["num_hit"] > 100
    assert out["stats"][1]["num_hit"] == 0 and out["stats"][2]["num_hit"] == 0
    # brick faces on lattice samples: the centre ray runs along z from the box face, so s0 + 16 m * h are the brick faces; a block of
    # voxels off the axis near the camera stretches the box, leaving empty bricks on the way to the plane
    g = tr.plane_grid((0, 0, 1), 0.6)
    blk = np.stack(np.meshgrid(np.arange(9, 12), np.arange(9, 12), np.arange(10, 13), indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    m = len(blk)
    g2 = dict(xyz=np.concatenate([g["xyz"], blk]), voxel_size=g["voxel_size"])
    for k in ("sdf0", "sdf_refined", "albedo"):
        g2[k] = np.concatenate([g[k], np.full(m, 0.02)])
    g2["weight"] = np.concatenate([g["weight"], np.ones(m, np.float32)])
    g2["rgb"] = np.concatenate([g["rgb"], np.full((m, 3), 50, np.uint8)])
    e = _constructed_engine(g2, [[0, 0, 0, 0, 0, 0]], W=33, H=27)
    out = _check_constructed(e, [0])
    assert out["stats"][0]["num_hit"] > 100
    na, nb = _skip_same(e, [0])
    assert na < nb, (na, nb)


def test_batch_single_repeat_and_engines_identical(tiny_scene):
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    engines = [Engine(0), Engine(0)]
    for e in engines:
        e.load_scene(s)
    batch = engines[0].render_keyframes([1, 3, 4])
    alone = engines[0].render_keyframes([3])
    for p in ALL:
        assert alone[p][0].tobytes() == batch[p][1].tobytes(), p
    assert alone["stats"][0] == batch["stats"][1]
    again = engines[0].render_keyframes([1, 3, 4])
    other = engines[1].render_keyframes([1, 3, 4])
    assert _bytes(batch) == _bytes(again) == _bytes(other)
    stats_only = engines[1].render_keyframes([1, 3, 4], planes=())
    assert set(stats_only) == {"stats"} and stats_only["stats"] == batch["stats"]


def test_after_prune_and_upsample(tiny_scene):
    """the brick bitmap and box are rebuilt for the new voxel set"""
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    vs = float(s["voxel_size"])
    e = Engine(0)
    e.load_scene(s)
    e.render_keyframes([0])
    e.clear_voxels_outside_thin_shell(vs)
    assert e.L.i3d_download_render(e.h, None, None, None, None, None) != 0
    assert "no render" in e.L.i3d_last_error(e.h).decode()
    e.set_sh(np.tile(s["sh"][0], (e.n, 1)))
    _check(e, [0, 4])
    e.upsample_grid()
    e.set_sh(np.tile(s["sh"][0], (e.n, 1)))
    out, _ = _check(e, [0, 4])
    _skip_same(e, [0, 4])
    assert out["stats"][0]["num_hit"] > 1000


def _gn_params(s):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    return p


def test_gn_iteration_unchanged_by_render(tiny_scene):
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    out = []
    for render in (False, True):
        e = Engine(0)
        e.load_scene(s)
        e.gn_iteration(_gn_params(s))
        if render:
            e.render_keyframes([0, 1, 2, 3, 4, 5])
            e.render_keyframes([2], "fused", ("depth",), False)
        info = e.gn_iteration(_gn_params(s))
        out.append((bytes(info)[:type(info).time_add.offset], e.download_state()))
    assert out[0][0] == out[1][0]
    for k in out[0][1]:
        assert out[0][1][k].tobytes() == out[1][1][k].tobytes(), k


def test_refusals_leave_engine_usable(tiny_scene):
    from intrinsic3d_b200.ctypes_defs import I3DRenderParams, I3DRenderStats
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    e = Engine(0)
    st = (I3DRenderStats * 4)()

    def refuse(ids, prm, text):
        a = np.ascontiguousarray(ids, np.int32)
        assert e.L.i3d_render_keyframes(e.h, len(a), a.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(prm), st) != 0
        assert text in e.L.i3d_last_error(e.h).decode(), e.L.i3d_last_error(e.h).decode()

    ok = I3DRenderParams(1, 31, 1, 0)
    refuse([0], ok, "no grid")
    n = len(s["xyz"])
    e.upload_grid(s["xyz"], s["sdf0"], s["sdf_refined"], s["albedo"], s["weight"], s["rgb"], s["voxel_size"])
    refuse([0], ok, "no frames")
    e.upload_frames(s["lum"], s["depth"])
    refuse([0], ok, "camera")
    e.set_camera(s["poses"], s["intr"], s["dist"])
    refuse([0], ok, "SH")
    refuse([0], I3DRenderParams(1, 1, 1, 0), "SH")
    e.set_sh(s["sh"])
    # (world > 1 is refused before any of these, as fusion does; a one-GPU test cannot reach it)
    refuse([], ok, "n > 0")
    refuse([0, 6], ok, "out of range")
    refuse([-1], ok, "out of range")
    for bad in (-1, 2):
        refuse([0], I3DRenderParams(bad, 31, 1, 0), "sdf_source")
    refuse([0], I3DRenderParams(1, 32, 1, 0), "planes")
    refuse([0], I3DRenderParams(1, -1, 1, 0), "planes")
    refuse([0], I3DRenderParams(1, 8, 0, 0), "photometric")
    refuse([0], I3DRenderParams(1, 1, 2, 0), "photometric")
    assert e.L.i3d_download_render(e.h, None, None, None, None, None) != 0
    with pytest.raises(ValueError):
        e.render_keyframes([0], "sdf0")
    with pytest.raises(ValueError):
        e.render_keyframes([0], planes=("colour",))
    out = e.render_keyframes([0], planes=("depth",), photometric=False)
    assert out["stats"][0]["num_hit"] > 1000 and out["stats"][0]["photo_count"] == 0
    buf = np.empty((1, 120, 160), np.float32)
    assert e.L.i3d_download_render(e.h, None, None, buf.ctypes.data_as(C.POINTER(C.c_float)), None, None) != 0
    assert "albedo plane was not rendered" in e.L.i3d_last_error(e.h).decode()
    e.upload_frames(s["lum"], s["depth"])                    # new frames drop the render
    assert e.L.i3d_download_render(e.h, None, None, None, None, None) != 0
    refuse(np.zeros(65536, np.int32), ok, "65535")
    # intrinsics that are not finite with fx, fy > 0, or distortion that is not finite (checked after pyr_scale)
    for intr, dist in (([0.0, 131.25, 79.5, 59.5], s["dist"]), ([131.25, -1.0, 79.5, 59.5], s["dist"]), ([131.25, 131.25, np.nan, 59.5], s["dist"]),
                       ([np.inf, 131.25, 79.5, 59.5], s["dist"])):
        e.set_camera(s["poses"], np.array(intr), dist)
        refuse([0], ok, "finite intrinsics")
    e.set_camera(s["poses"], s["intr"], np.array([0.0, np.nan, 0.0, 0.0, 0.0]))
    refuse([0], ok, "distortion")
    e.set_camera(s["poses"], s["intr"], s["dist"])
    e.upload_frames(s["lum"], s["depth"], 0.0)              # pyramid scale 0: fx = fy = 0
    refuse([0], ok, "finite intrinsics")
    e.upload_frames(s["lum"], s["depth"])
    e.upsample_grid()                                       # a new voxel set drops the per-voxel SH
    refuse([0], ok, "SH")
    e.set_sh(np.tile(s["sh"][0], (e.n, 1)))
    assert n < e.n
    _check(e, [0, 5])


def test_non_finite_pose_renders_no_hit(tiny_scene):
    """A NaN or infinite pose: that view has no hit (its march ends at once), the others are unaffected, all byte-equal to the restatement"""
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    e = Engine(0)
    e.load_scene(s)
    want = e.render_keyframes([0, 3])
    poses = s["poses"].copy()
    poses[1, 0] = np.nan
    poses[2, 4] = np.inf
    e.set_camera(poses, s["intr"], s["dist"])
    for skip in (True, False):
        e.set_render_skip(skip)
        out, _ = _check(e, [0, 1, 2, 3])
        for i in (1, 2):
            assert out["stats"][i]["num_hit"] == 0 and not out["depth"][i].any() and out["stats"][i]["num_observed"] > 0
        for p in ALL:
            assert out[p][[0, 3]].tobytes() == want[p].tobytes(), p
        assert [out["stats"][i] for i in (0, 3)] == want["stats"]


def test_c2_statistics_skip_on_off():
    """C2 (~500 K voxels, 50 keyframes at 640 x 480), statistics only: skipping changes nothing but the samples evaluated"""
    import torch
    from intrinsic3d_b200.engine import Engine
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c2", device="cuda" if torch.cuda.is_available() else "cpu")
    e = Engine(0)
    e.load_scene(s)
    ids = list(range(s["depth"].shape[0]))
    runs = []
    for skip in (True, False, True):
        e.set_render_skip(skip)
        out = e.render_keyframes(ids, planes=())
        runs.append((out["stats"], e.phase_count("render_samples"), e.phase_ms("render")))
    assert runs[0][0] == runs[1][0] == runs[2][0]
    assert runs[0][1] == runs[2][1] < runs[1][1]
    assert all(st["depth_count"] > 10000 for st in runs[0][0])
    print("samples skip/dense", runs[0][1], runs[1][1], "ms", runs[2][2], runs[1][2])
