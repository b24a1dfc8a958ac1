"""GPU tests of frame-to-model tracking (i3d_track_sensor_frames) against the restatement tests/track_ref.py: pyramid, normals, prediction
planes and correspondence masks byte-equal, counts exact, sums to 1e-12 relative; the tiny scene's accuracy gates of tests/test_track.py,
C2 fused from the store, byte identity across calls, engines, batches and chunks, the refusals, and the state a call must leave alone."""
import ctypes as C
import os

import numpy as np
import pytest

import render_ref as rr
import track_ref as tr
from test_track import check_kt3, kt3_cases

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _engine(grid, depth, dcam, copies=1):
    """an engine holding `grid` (dict of the scene arrays) and the depth frames in its sensor store (`copies` times over)"""
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.upload_grid(grid["xyz"], grid["sdf0"], grid["sdf_refined"], grid["albedo"], grid["weight"], grid["rgb"], float(grid["voxel_size"]))
    depth = np.ascontiguousarray(np.concatenate([depth] * copies), np.float32)
    F, H, W = depth.shape
    e.sensor_frames_begin(dcam, dcam, F)
    e.sensor_frames_add(depth, np.zeros((F, H, W, 3), np.uint8))
    return e


def _dcam(s):
    F, H, W = s["depth"].shape
    return (W, H) + tuple(float(v) for v in s["intr"])


def _rel(a, b, rel=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.all(np.abs(a - b) <= rel * np.maximum(np.abs(b), 1e-300))


def _compare(e, frames, ids, poses, levels, planes=True, pose_tol=1e-12):
    """the engine's last call against restated Frames: planes of the last pass, sums, outcome and poses"""
    n = len(ids)
    sums, T = e.debug_track_system(n)
    for k, f in enumerate(frames):
        assert f.sys[28] == sums[k, 28] and _rel(sums[k], f.sys), (k, sums[k], f.sys)
        assert [f.status, f.iterations] == [poses[1][k]["status"], poses[1][k]["iterations"]], (k, f.status, poses[1][k])
        assert f.correspondences == poses[1][k]["correspondences"]
        assert np.abs(np.array(f.w2c) - poses[0][k]).max() <= pose_tol
        assert np.abs(np.array(f.T) - T[k]).max() <= pose_tol
    if planes:
        for l in range(levels):
            P = e.debug_track_planes(l, n)
            for k, f in enumerate(frames):
                assert P["depth"][k].tobytes() == f.depth[l].tobytes(), ("depth", l, k)
                assert P["normal"][k].tobytes() == f.nrm[l].tobytes(), ("normal", l, k)
                if l == 0:
                    assert P["pred_depth"][k].tobytes() == f.pdepth.tobytes(), ("pred_depth", k)
                    assert P["pred_normal"][k].tobytes() == f.pnrm.tobytes(), ("pred_normal", k)
                    assert P["mask"][k].tobytes() == f.mask.tobytes(), ("mask", k, int((P["mask"][k] != f.mask).sum()))


def _initial_same(info, f):
    st = info["initial"]
    for k in ("num_hit", "num_observed", "depth_count"):
        assert st[k] == f.initial[k], (k, st[k], f.initial[k])
    for k in ("depth_abs", "depth_sq"):
        assert abs(st[k] - f.initial[k]) <= 1e-12 * max(abs(f.initial[k]), 1e-300)


@pytest.mark.parametrize("source", ["fused", "refined"])
def test_planes_masks_and_level0_system_at_input_pose(tiny_scene, source):
    s = tiny_scene
    dcam = _dcam(s)
    e = _engine(s, s["depth"], dcam)
    ids = [0, 2, 5]
    pose_in = tr.aa_to_rt(s["poses"])[ids]
    out = e.track_sensor_frames(ids, pose_in, source, num_levels=3, iterations=(0, 0, 0))
    g = rr.Grid(s["xyz"], s["sdf0"] if source == "fused" else s["sdf_refined"], s["albedo"], s["weight"], s["voxel_size"])
    p = tr.params(num_levels=3, iterations=(0, 0, 0))
    frames = [tr.Frame(s["depth"][f], pose_in[k], dcam, p, grid=g).run() for k, f in enumerate(ids)]
    _compare(e, frames, ids, out, 3)
    assert np.array_equal(out[0], pose_in)                          # no iteration: the input pose comes back unchanged
    for info, f in zip(out[1], frames):
        _initial_same(info, f)
        assert info["correspondences"] > 3000
    assert e.phase_ms("track") > 0 and e.phase_count("track_correspondences") == sum(f.correspondences for f in frames)


def test_one_iteration_exact(tiny_scene):
    s = tiny_scene
    dcam = _dcam(s)
    e = _engine(s, s["depth"], dcam)
    ids = [3, 1]
    pose_in = tr.aa_to_rt(s["poses"])[ids]
    out = e.track_sensor_frames(ids, pose_in, "fused", num_levels=1, iterations=(1,))
    g = rr.Grid(s["xyz"], s["sdf0"], s["albedo"], s["weight"], s["voxel_size"])
    p = tr.params(num_levels=1, iterations=(1,))
    frames = [tr.Frame(s["depth"][f], pose_in[k], dcam, p, grid=g).run() for k, f in enumerate(ids)]
    _compare(e, frames, ids, out, 1)
    assert all(i["iterations"] == 1 and i["status"] == 0 and i["update_norm"] > 0 for i in out[1])


@pytest.mark.parametrize("source", ["fused", "refined"])
def test_full_schedule_tiny_scene(tiny_scene, source):
    s = tiny_scene
    dcam = _dcam(s)
    F = s["depth"].shape[0]
    e = _engine(s, s["depth"], dcam)
    g = rr.Grid(s["xyz"], s["sdf0"] if source == "fused" else s["sdf_refined"], s["albedo"], s["weight"], s["voxel_size"])
    true, cases = kt3_cases(s)
    for name, start in cases.items():
        out = e.track_sensor_frames(list(range(F)), start, source)
        frames = tr.track(g, s["depth"], list(range(F)), start, dcam)
        _compare(e, frames, list(range(F)), out, 3, planes=False, pose_tol=1e-6)
        r, t = check_kt3(name, start, out[0], true)
        print(source, name, "rot deg", np.round(r, 4), "centre mm", np.round(t * 1e3, 4), "device ms", e.phase_ms("track"))


def test_golden_fixture_on_device():
    g = np.load(os.path.join(HERE, "golden", "tiny_track.npz"))
    dcam = tuple(g["dcam"].tolist())
    e = _engine(g, g["depth"], dcam)
    ids = g["ids"].tolist()
    out = e.track_sensor_frames(ids, g["pose_in"], "fused", num_levels=int(g["num_levels"]), iterations=g["iterations"].tolist())
    sums, _ = e.debug_track_system(len(ids))
    assert _rel(sums, g["sums"])
    assert [[i["status"], i["iterations"], i["correspondences"]] for i in out[1]] == g["outcome"].tolist()
    assert np.abs(out[0] - g["pose_out"]).max() < 1e-12
    for l in range(int(g["num_levels"])):
        P = e.debug_track_planes(l, len(ids))
        assert P["depth"].tobytes() == g[f"depth_{l}"].tobytes() and P["normal"].tobytes() == g[f"normal_{l}"].tobytes()
    assert P["pred_depth"].tobytes() == g["pred_depth"].tobytes() and P["pred_normal"].tobytes() == g["pred_normal"].tobytes()
    assert P["mask"].tobytes() == g["mask"].tobytes()


def _bytes(out):
    return out[0].tobytes() + repr(out[1]).encode()


def test_byte_identity_calls_engines_batches_chunks(tiny_scene):
    s = tiny_scene
    dcam = _dcam(s)
    F = s["depth"].shape[0]
    copies = 7                                                        # 42 stored frames: two passes of I3D_TRACK_CHUNK = 32
    A = _engine(s, s["depth"], dcam, copies)
    B = _engine(s, s["depth"], dcam, copies)
    n = F * copies
    start = np.concatenate([tr.perturb(tr.aa_to_rt(s["poses_true"]), 1.0, 0.01, seed=9 + c) for c in range(copies)])
    ids = list(range(n))
    a1 = A.track_sensor_frames(ids, start)
    a2 = A.track_sensor_frames(ids, start)
    b1 = B.track_sensor_frames(ids, start)
    assert _bytes(a1) == _bytes(a2) == _bytes(b1)
    rev = B.track_sensor_frames(ids[::-1], start[::-1])
    assert rev[0][::-1].tobytes() == a1[0].tobytes() and rev[1][::-1] == a1[1]
    for k in (0, 31, 32, 41):                                         # alone, and on both sides of the chunk boundary
        one = B.track_sensor_frames([k], start[k:k + 1])
        assert one[0].tobytes() == a1[0][k:k + 1].tobytes() and one[1][0] == a1[1][k], k
    # frames 33.. of a call that starts at frame 1 land in the first chunk instead of the second
    sh = B.track_sensor_frames(ids[1:], start[1:])
    assert sh[0].tobytes() == a1[0][1:].tobytes() and sh[1] == a1[1][1:]


def test_c2_fused_from_store_tracks_every_frame():
    from fusion_ref import depth_range, scene_inputs
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene
    import torch
    s = config_scene("c2", device="cuda:0" if torch.cuda.is_available() else "cpu")
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    F = depth.shape[0]
    e = engine.Engine(0)
    e.sensor_frames_begin(dcam, ccam, F)
    e.sensor_frames_add(depth, bgr)
    p = engine.default_fusion_params()
    p.voxel_size = float(s["voxel_size"])
    p.depth_min, p.depth_max = depth_range(s)
    e.fusion_begin(p)
    ids = np.arange(F, dtype=np.int32)
    e.fusion_integrate_sensor(ids, c2w, w2c)
    assert e.fusion_finish() > 100000
    true = tr.aa_to_rt(s["poses_true"])
    start = tr.perturb(true, 0.5, 0.005, seed=21)
    out, infos = e.track_sensor_frames(ids, start, "fused")
    r0, t0 = tr.pose_errors(start, true)
    r1, t1 = tr.pose_errors(out, true)
    print("C2 rot deg", r1.max(), np.median(r1), "centre mm", 1e3 * t1.max(), 1e3 * np.median(t1), "device ms", e.phase_ms("track"))
    assert all(i["status"] == 0 for i in infos)
    assert (t1 * 10 <= t0).all(), (t0, t1)
    assert (r1 < r0).all(), (r0, r1)


def _refused(e, fn, text):
    with pytest.raises(RuntimeError, match=text):
        fn()


def test_refusals_and_untouched_state(tiny_scene):
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    dcam = _dcam(s)
    F = s["depth"].shape[0]
    pose = tr.aa_to_rt(s["poses"])
    # no grid, no store
    e0 = Engine(0)
    _refused(e0, lambda: e0.track_sensor_frames([0], pose[:1]), "no grid")
    e0.upload_grid(s["xyz"], s["sdf0"], s["sdf_refined"], s["albedo"], s["weight"], s["rgb"], s["voxel_size"])
    _refused(e0, lambda: e0.track_sensor_frames([0], pose[:1]), "no frames in the sensor store")
    e = _engine(s, s["depth"], dcam)
    bad = pose[:2].copy(); bad[1, 4] = np.nan
    L = e.L
    cases = [
        (lambda: e.track_sensor_frames([], pose[:0]), "n > 0"),
        (lambda: e.track_sensor_frames([0, F], pose[:2]), "out of range"),
        (lambda: e.track_sensor_frames([-1], pose[:1]), "out of range"),
        (lambda: e.track_sensor_frames([1, 1], pose[:2]), "repeated"),
        (lambda: e.track_sensor_frames([0, 1], bad), "not finite"),
        (lambda: e.track_sensor_frames([0], pose[:1], num_levels=0), "num_levels"),
        (lambda: e.track_sensor_frames([0], pose[:1], num_levels=5), "num_levels"),
        (lambda: e.track_sensor_frames([0], pose[:1], iterations=(1, -1, 0)), "negative"),
        (lambda: e.track_sensor_frames([0], pose[:1], max_distance=0.0), "max_distance"),
        (lambda: e.track_sensor_frames([0], pose[:1], max_distance=float("inf")), "max_distance"),
        (lambda: e.track_sensor_frames([0], pose[:1], min_normal_cos=1.5), "min_normal_cos"),
        (lambda: e.track_sensor_frames([0], pose[:1], min_normal_cos=float("nan")), "min_normal_cos"),
        (lambda: e.track_sensor_frames([0], pose[:1], min_correspondences=5), "min_correspondences"),
    ]
    for fn, text in cases:
        _refused(e, fn, text)
    p = engine.default_track_params()
    p.sdf_source = 2
    out = np.empty((1, 12)); ids = np.zeros(1, np.int32); pin = np.ascontiguousarray(pose[:1])
    assert L.i3d_track_sensor_frames(e.h, 1, ids.ctypes.data_as(C.POINTER(C.c_int32)), pin.ctypes.data_as(C.POINTER(C.c_double)), C.byref(p),
                                     out.ctypes.data_as(C.POINTER(C.c_double)), None) != 0
    assert b"sdf_source" in L.i3d_last_error(e.h)
    _refused(e, lambda: e.debug_track_system(1), "no tracking call")
    # a level built from a level under 3 px
    small = np.zeros((1, 10, 12), np.float32)
    es = _engine(s, small, (12, 10, 10.0, 10.0, 6.0, 5.0))
    _refused(es, lambda: es.track_sensor_frames([0], pose[:1], num_levels=4), "at least 3 px")
    es.track_sensor_frames([0], pose[:1], num_levels=3, iterations=(0, 0, 0))
    # usable afterwards
    a = e.track_sensor_frames([0, 1], pose[:2])
    assert all(i["status"] == 0 for i in a[1])


def test_refinement_render_and_mesh_unchanged_by_tracking(tiny_scene):
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    dcam = _dcam(s)
    F = s["depth"].shape[0]

    def run(track):
        e = Engine(0)
        e.load_scene(s)
        e.sensor_frames_begin(dcam, dcam, F)
        e.sensor_frames_add(s["depth"], np.zeros(s["depth"].shape + (3,), np.uint8))
        e.render_keyframes([0, 3])
        m = e.extract_mesh("refined")
        if track:
            e.track_sensor_frames(list(range(F)), tr.aa_to_rt(s["poses"]), "refined")
        W, H = e.frame_size
        planes = [np.empty((2, H, W), np.float32), np.empty((2, H, W, 3), np.float32)] + [np.empty((2, H, W), np.float32) for _ in range(3)]
        e._check(e.L.i3d_download_render(e.h, *(pl.ctypes.data_as(C.POINTER(C.c_float)) for pl in planes)))
        mesh = [np.empty_like(m["vertices"]), np.empty_like(m["colors"]), np.empty_like(m["faces"])]
        e._check(e.L.i3d_download_mesh(e.h, mesh[0].ctypes.data_as(C.POINTER(C.c_float)), mesh[1].ctypes.data_as(C.POINTER(C.c_uint8)),
                                       mesh[2].ctypes.data_as(C.POINTER(C.c_int32))))
        info = {k: v for k, v in e.gn_iteration(engine.default_params()).as_dict().items() if not k.startswith("time_")}
        st = e.download_state()
        return b"".join(pl.tobytes() for pl in planes), b"".join(a.tobytes() for a in mesh), \
            repr(info) + b"".join(np.asarray(v).tobytes() for v in st.values()).hex()
    a, b = run(False), run(True)
    assert a[0] == b[0], "render planes changed"
    assert a[1] == b[1], "resident mesh changed"
    assert a[2] == b[2], "GN iteration changed"
