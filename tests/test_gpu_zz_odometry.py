"""GPU tests of tracking against the fusion in progress (i3d_fusion_track_sensor_frames) and of dense RGB-D odometry
(i3d_fusion_track_and_integrate_sensor), DESIGN.md §6o: byte identity with i3d_fusion_finish(correct 0) + i3d_track_sensor_frames, the loop
frame by frame against the restatement of tests/test_odometry.py, the golden fixture, byte identity across calls, engines and chunks,
accuracy on C2 geometry (first 25 frames: see that test), the refusals and the pipeline after the loop."""
import ctypes as C

import numpy as np
import pytest

import track_ref as tr
from fusion_ref import depth_range, scene_inputs
from test_odometry import ANCHORED, Odometry, dense_tiny
from test_gpu_zz_track import _rel

pytestmark = pytest.mark.gpu


def _engine(s, correct=0):
    """an engine with the scene's frames in its sensor store and a fusion begun with the scene's voxel size and depth range"""
    from intrinsic3d_b200 import engine
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    e = engine.Engine(0)
    e.sensor_frames_begin(dcam, ccam, depth.shape[0])
    e.sensor_frames_add(depth, bgr)
    p = engine.default_fusion_params()
    p.voxel_size = float(s["voxel_size"])
    p.depth_min, p.depth_max = depth_range(s)
    p.correct_sdf_iterations = correct
    e.fusion_begin(p)
    return e, c2w, w2c


def _volume_bytes(e):
    v = e.fusion_volume()
    return b"".join(v[k].tobytes() for k in ("xyz", "sdf", "weight", "rgb"))


def _planes(e, n, levels):
    return [e.debug_track_planes(l, n) for l in range(levels)]


@pytest.mark.parametrize("skip", [True, False])
def test_identity_with_finish_and_track(skip):
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    for k in (1, 3, 10):
        e, c2w, w2c = _engine(s)
        e.set_render_skip(skip)
        e.fusion_integrate_sensor(np.arange(k), c2w[:k], w2c[:k])
        ids = [k, k + 1, k + 2]
        start = tr.perturb(true[ids], 1.0, 0.005, seed=k)
        vol = _volume_bytes(e)
        live = e.fusion_track_sensor_frames(ids, start)
        live_sys = e.debug_track_system(3)
        live_planes = _planes(e, 3, 3)
        assert _volume_bytes(e) == vol, "the live call changed the fusion volume"
        assert e.phase_ms("track") > 0 and e.phase_ms("track_bricks") > 0
        assert e.fusion_finish() > 0
        fin = e.track_sensor_frames(ids, start, "fused")
        fin_sys = e.debug_track_system(3)
        fin_planes = _planes(e, 3, 3)
        assert live[0].tobytes() == fin[0].tobytes() and live[1] == fin[1], (k, skip)
        assert live_sys[0].tobytes() == fin_sys[0].tobytes() and live_sys[1].tobytes() == fin_sys[1].tobytes()
        for a, b in zip(live_planes, fin_planes):
            for name in a:
                assert a[name].tobytes() == b[name].tobytes(), (k, skip, name)
        print("identity", k, skip, [i["status"] for i in live[1]], [i["initial"]["num_hit"] for i in live[1]])


def test_loop_frame_by_frame_against_the_restatement():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e, _, _ = _engine(s)
    odo = Odometry(s, iterations=(4, 2, 2))
    motion = []                                        # the device's integrated camera -> world poses
    for f in range(8):
        first = true[0] if f == 0 else None
        out, info = e.fusion_track_and_integrate_sensor([f], first, iterations=(4, 2, 2))
        st, w, frame = odo.step(f, pose_first=first, motion=None if f == 0 else motion)
        assert info[0]["status"] == st, (f, info[0]["status"], st)
        assert np.abs(out[0] - w).max() <= 1e-12, f
        if st == ANCHORED:
            motion = [tr.inverse(true[0])]
        else:
            sums, T = e.debug_track_system(1)
            assert sums[0, 28] == frame.sys[28] and _rel(sums[0], frame.sys), f
            assert np.abs(T[0] - np.array(frame.T)).max() <= 1e-12
            motion = (motion + [list(T[0])])[-2:]
        v = e.fusion_volume()
        o = odo.volume()
        for k in ("xyz", "sdf", "weight", "rgb"):
            assert v[k].tobytes() == o[k].tobytes(), (f, k)
    assert e.phase_ms("odometry") > 0 and e.phase_ms("odometry_predict") > 0 and e.phase_ms("odometry_icp") > 0


def test_golden_fixture_on_device():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_odometry.npz"))
    s = dense_tiny(int(g["frames"]))
    e, _, _ = _engine(s)
    out, info = e.fusion_track_and_integrate_sensor(g["ids"], g["pose_first"], iterations=tuple(g["iterations"].tolist()))
    assert [i["status"] for i in info] == g["status"].tolist()
    assert np.abs(out - g["pose_out"]).max() <= 1e-12
    v = e.fusion_volume()
    for k in ("xyz", "sdf", "weight", "rgb"):
        assert v[k].tobytes() == g[f"volume_{k}"].tobytes(), k


def _run(s, ids, first, chunks):
    e, _, _ = _engine(s)
    outs = []
    for c, part in enumerate(np.array_split(np.asarray(ids, np.int32), chunks)):
        outs.append(e.fusion_track_and_integrate_sensor(part, first if c == 0 else None))
    poses = np.concatenate([o[0] for o in outs])
    infos = [i for o in outs for i in o[1]]
    return poses.tobytes() + repr(infos).encode(), _volume_bytes(e)


def test_byte_identity_calls_engines_chunks():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    ids = [k % 72 for k in range(200)]                 # the orbit is periodic: frame 0 follows frame 71
    a = _run(s, ids, true[0], 1)
    b = _run(s, ids, true[0], 1)
    c = _run(s, ids, true[0], 4)
    assert a == b == c


def test_c2_accuracy_first_25_of_200_frames():
    """C2 geometry, 200 frames (2.5 deg of orbit per frame), frame 0 anchored at its true pose.  Measured on an H100: the first 21 tracked
    frames stay within 0.015 deg and 0.12 mm; from about frame 22 the rotation about the sphere's centre, constrained only by its 3 %
    bumps, grows by about 1.5x per frame (0.04 deg at frame 25, 2 deg at 34) and tracking is lost at frame 40 (status 1 from there).  So
    the proposed gates (camera centre <= 2 mm, rotation <= 0.2 deg, median |dsdf| <= 0.1 voxel) are checked on the first 25 frames only."""
    import torch
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c2", device="cuda:0" if torch.cuda.is_available() else "cpu", frames=200)
    true = tr.aa_to_rt(s["poses_true"])
    e, c2w, w2c = _engine(s)
    ids = np.arange(25, dtype=np.int32)
    out, info = e.fusion_track_and_integrate_sensor(ids, true[0])
    st = [i["status"] for i in info]
    r, t = tr.pose_errors(out, true[ids])
    print("C2 odometry, 25 frames: rot deg max %.4f median %.4f, centre mm max %.4f median %.4f, wall ms %.1f" %
          (r.max(), np.median(r), 1e3 * t.max(), 1e3 * np.median(t), e.phase_ms("odometry")))
    tracked = e.fusion_volume()
    ref, _, _ = _engine(s)
    ref.fusion_integrate_sensor(ids, c2w[ids], w2c[ids])
    fused = ref.fusion_volume()
    ka, kb = tracked["weight"] > 0, fused["weight"] > 0
    A = {tuple(x): i for i, x in enumerate(tracked["xyz"][ka])}
    common = [(A[tuple(x)], j) for j, x in enumerate(fused["xyz"][kb]) if tuple(x) in A]
    ia, ib = np.array([c[0] for c in common]), np.array([c[1] for c in common])
    overlap = len(common) / max(ka.sum(), kb.sum())
    dsdf = np.abs(tracked["sdf"][ka][ia].astype(np.float64) - fused["sdf"][kb][ib]) / float(s["voxel_size"])
    print("C2 grid, 25 frames: voxel overlap %.4f, median |dsdf| %.4f voxel" % (overlap, np.median(dsdf)))
    assert st[0] == ANCHORED and all(x == 0 for x in st[1:]), st
    assert t.max() <= 0.002 and r.max() <= 0.2, (r.max(), t.max())
    assert np.median(dsdf) <= 0.1


def _refused(fn, text):
    with pytest.raises(RuntimeError, match=text):
        fn()


def test_refusals_leave_everything_as_it_was():
    from intrinsic3d_b200 import engine
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e0 = engine.Engine(0)
    _refused(lambda: e0.fusion_track_and_integrate_sensor([0], true[0]), "no fusion in progress")
    e, c2w, w2c = _engine(s)
    _refused(lambda: e.fusion_track_sensor_frames([0], true[:1]), "no voxel with weight > 0")
    _refused(lambda: e.fusion_track_and_integrate_sensor([0]), "motion state")
    e.fusion_integrate_sensor([0, 1], c2w[:2], w2c[:2])
    bad = true[:2].copy(); bad[1, 3] = np.inf
    vol = _volume_bytes(e)
    cases = [
        (lambda: e.fusion_track_sensor_frames([], true[:0]), "n > 0"),
        (lambda: e.fusion_track_sensor_frames([0, 72], true[:2]), "out of range"),
        (lambda: e.fusion_track_sensor_frames([1, 1], true[:2]), "repeated"),
        (lambda: e.fusion_track_sensor_frames([0, 1], bad), "not finite"),
        (lambda: e.fusion_track_sensor_frames([0], true[:1], num_levels=5), "num_levels"),
        (lambda: e.fusion_track_sensor_frames([0], true[:1], min_correspondences=5), "min_correspondences"),
        (lambda: e.fusion_track_and_integrate_sensor([0], bad[1]), "pose_first of entry 0 is not finite"),
        (lambda: e.fusion_track_and_integrate_sensor([0]), "motion state"),       # an integrate call cleared it
        (lambda: e.fusion_track_and_integrate_sensor([-1], true[0]), "out of range"),
        (lambda: e.fusion_track_and_integrate_sensor([0], true[0], iterations=(1, -1)), "negative"),
        (lambda: e.fusion_track_and_integrate_sensor([0], true[0], max_distance=0.0), "max_distance"),
    ]
    for fn, text in cases:
        _refused(fn, text)
        assert _volume_bytes(e) == vol
    p = engine.default_track_params()
    p.sdf_source = 1
    out = np.empty((1, 12)); ids = np.zeros(1, np.int32); pin = np.ascontiguousarray(true[:1])
    for fn in (e.L.i3d_fusion_track_sensor_frames, e.L.i3d_fusion_track_and_integrate_sensor):
        assert fn(e.h, 1, ids.ctypes.data_as(C.POINTER(C.c_int32)), pin.ctypes.data_as(C.POINTER(C.c_double)), C.byref(p),
                  out.ctypes.data_as(C.POINTER(C.c_double)), None) != 0
        assert b"sdf_source" in e.L.i3d_last_error(e.h)
    assert _volume_bytes(e) == vol
    # the fusion is still in progress and usable
    out, info = e.fusion_track_and_integrate_sensor([2, 3], true[2])
    assert [i["status"] for i in info] == [0, 0]
    out, info = e.fusion_track_and_integrate_sensor([4])                  # continues from the motion state
    assert info[0]["status"] == 0


def test_pipeline_finish_and_mesh_after_the_loop():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e, _, _ = _engine(s, correct=10)
    out, info = e.fusion_track_and_integrate_sensor(list(range(24)), true[0])
    assert all(i["status"] == 0 for i in info[1:])
    assert e.fusion_finish() > 1000
    m = e.extract_mesh("fused")
    assert len(m["faces"]) > 100
