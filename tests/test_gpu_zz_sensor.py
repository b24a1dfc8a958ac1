"""GPU checks of the sensor store (i3d_sensor_frames_begin / add, i3d_sensor_keyframe_scores, i3d_fusion_integrate_sensor,
i3d_select_rgbd_frames): the resized keyframes byte-equal to tests/sensor_ref.py, and every consumer of the store byte-identical to the same
work fed from host buffers, up to a Gauss-Newton iteration of the whole chain."""
import ctypes as C

import numpy as np
import pytest

import frames_ref
import sensor_ref
from test_gpu_zz_fusion import CASES, _inputs, _params, _same, _scene

pytestmark = pytest.mark.gpu


def _engine():
    from intrinsic3d_b200.engine import Engine
    return Engine(0)


def _bgr(F, cam, seed):
    return np.random.default_rng(seed).integers(0, 256, (F, int(cam[1]), int(cam[0]), 3), dtype=np.uint8)


def _stored(dcam, depth, ccam, bgr, chunks=None):
    e = _engine()
    e.sensor_frames_begin(dcam, ccam, len(depth))
    for a, b in (chunks or [(0, len(depth))]):
        e.sensor_frames_add(depth[a:b], bgr[a:b])
    assert e.sensor_num_frames() == len(depth)
    return e


def _cams():
    s = _scene()
    dcam, depth = _inputs(s)[:2]
    return s, dcam, depth, sensor_ref.color_cameras(dcam)


@pytest.mark.parametrize("cam", ["color_x2", "same_size", "x1.5_shifted"])
def test_selected_planes_byte_equal_restatement(cam):
    s, dcam, depth, cams = _cams()
    ccam = cams[cam]
    bgr = _bgr(len(depth), ccam, seed=1)
    e = _stored(dcam, depth, ccam, bgr)
    ids = [3, 0, 4]
    e.select_rgbd_frames(ids)
    assert e.use_rgbd_level(0) == (ccam[0], ccam[1])
    lg, dg, cg = e.debug_frames(with_color=True)
    rd = sensor_ref.resize_depth(depth[ids], dcam, ccam)
    assert dg.tobytes() == rd.tobytes()
    assert lg.tobytes() == frames_ref.intensity0(bgr[ids]).tobytes()
    assert cg.tobytes() == bgr[ids].tobytes()
    if cam != "same_size":
        assert e.phase_ms("resize_depth") > 0
    if cam == "x1.5_shifted":                                   # taps outside the depth plane give 0
        assert (dg[:, :, :10] == 0).all() and (dg[:, -10:, :] == 0).all() and (dg > 0).sum() > 1000


def test_golden_fixture_on_device():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_sensor.npz"))
    dcam, ccam = tuple(g["depth_cam"]), tuple(g["color_cam"])
    dcam, ccam = (int(dcam[0]), int(dcam[1])) + dcam[2:], (int(ccam[0]), int(ccam[1])) + ccam[2:]
    e = _stored(dcam, g["depth"], ccam, _bgr(len(g["depth"]), ccam, seed=2))
    e.select_rgbd_frames([0, 1])
    e.use_rgbd_level(0)
    assert e.debug_frames()[1].tobytes() == g["resized"].tobytes()


def test_unsorted_repeated_ids_match_host_upload_at_every_level():
    s, dcam, depth, cams = _cams()
    ccam = cams["color_x2"]
    bgr = _bgr(len(depth), ccam, seed=3)
    ids = [4, 1, 1, 3, 0, 4]
    A = _stored(dcam, depth, ccam, bgr)
    A.select_rgbd_frames(ids)
    B = _engine()
    B.upload_rgbd_frames(bgr[ids], sensor_ref.resize_depth(depth[ids], dcam, ccam))
    for lvl in (0, 1, 2):
        assert A.use_rgbd_level(lvl) == B.use_rgbd_level(lvl)
        fa, fb = A.debug_frames(with_color=(lvl == 0)), B.debug_frames(with_color=(lvl == 0))
        for a, b in zip(fa, fb):
            assert (a is None and b is None) or a.tobytes() == b.tobytes(), lvl


def test_store_scores_equal_host_scores_across_adds():
    from intrinsic3d_b200.engine import KEYFRAME_CHUNK
    F = KEYFRAME_CHUNK + 5
    ccam, dcam = (96, 72, 80.0, 80.0, 47.5, 35.5), (48, 36, 40.0, 40.0, 23.5, 17.5)
    bgr = _bgr(F, ccam, seed=4)
    bgr[::3] = (bgr[::3] // 2 + 60).astype(np.uint8)
    bgr[2] = 77                                                  # a constant frame: NaN, as in the reference
    depth = np.random.default_rng(5).random((F, 36, 48)).astype(np.float32)
    e = _stored(dcam, depth, ccam, bgr, chunks=[(0, 10), (10, 30), (30, F)])
    got = e.sensor_keyframe_scores()
    assert e.phase_count("keyframe_chunks") == 2 and e.phase_ms("keyframe_scores") > 0
    ref = _engine().keyframe_scores(bgr)
    assert np.isnan(got[2]) and got.tobytes() == ref.tobytes()


def _fuse_store(p, inp, ids, e=None):
    dcam, depth, ccam, bgr, c2w, w2c = inp
    e = e or _stored(dcam, depth, ccam, bgr)
    e.fusion_begin(p)
    e.fusion_integrate_sensor(ids, c2w[ids], w2c[ids])
    return e


def _fuse_host(p, inp, ids):
    dcam, depth, ccam, bgr, c2w, w2c = inp
    e = _engine()
    e.fusion_begin(p)
    e.fusion_integrate(dcam, depth[ids], ccam, bgr[ids], c2w[ids], w2c[ids])
    return e


def _same_grid(a, b):
    ga, gb = a.download_grid(), b.download_grid()
    for k in ("xyz", "sdf0", "sdf_refined", "albedo", "weight", "rgb", "voxel_size"):
        assert np.asarray(ga[k]).tobytes() == np.asarray(gb[k]).tobytes(), k


@pytest.mark.parametrize("case", list(CASES))
def test_fusion_from_store_matches_host_frames(case):
    c = CASES[case]
    s = _scene()
    clip = (-1.0, 1.0, -1.0, 0.0, -1.0, 1.0) if c.get("clip") else None
    p = _params(s, window=c.get("window", 2), ws=c.get("ws", 10.0), clip=clip)
    inp = _inputs(s, frames=c.get("frames"), color_x2=c.get("color_x2", False))
    ids = list(range(len(inp[1])))
    A, B = _fuse_store(p, inp, ids), _fuse_host(p, inp, ids)
    _same(A.fusion_volume(), B.fusion_volume())
    assert A.fusion_finish() == B.fusion_finish() > 1000
    _same_grid(A, B)


def test_fusion_from_store_subset_growth_and_store_unchanged():
    s = _scene()
    inp = _inputs(s, color_x2=True)
    ids = [3, 0, 4, 1]
    p = _params(s, cap=1024)
    A, B = _fuse_store(p, inp, ids), _fuse_host(p, inp, ids)
    assert A.phase_count("fusion_growths") >= 3 and A.phase_count("fusion_growths") == B.phase_count("fusion_growths")
    _same(A.fusion_volume(), B.fusion_volume())
    A.fusion_finish(), B.fusion_finish()
    _same_grid(A, B)
    first = A.download_grid()
    _fuse_store(p, inp, ids, A)                                  # the same store again: erosion did not write into it
    A.fusion_finish()
    second = A.download_grid()
    for k in first:
        assert np.asarray(first[k]).tobytes() == np.asarray(second[k]).tobytes(), k


def _info_bytes(info):
    return bytes(info)[:type(info).time_add.offset]             # every I3DIterInfo field before the wall-clock timers


def test_whole_chain_from_one_upload_matches_host_chain():
    """scores -> select_keyframes -> fuse the keyframes -> finish -> select -> level 1 -> lighting -> one GN iteration."""
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.ctypes_defs import default_params
    from intrinsic3d_b200.keyframes import select_keyframes
    s = _scene()
    dcam, depth, ccam, bgr, c2w, w2c = inp = _inputs(s, color_x2=True)
    p = _params(s)
    A, B = _stored(dcam, depth, ccam, bgr, chunks=[(0, 2), (2, len(depth))]), _engine()
    sa, sb = A.sensor_keyframe_scores(), B.keyframe_scores(bgr)
    assert sa.tobytes() == sb.tobytes()
    kf = np.nonzero(select_keyframes(sa, 2))[0]
    assert 2 <= len(kf) < len(depth)
    _fuse_store(p, inp, kf, A)
    B.fusion_begin(p)
    B.fusion_integrate(dcam, depth[kf], ccam, bgr[kf], c2w[kf], w2c[kf])
    assert A.fusion_finish() == B.fusion_finish() > 1000
    A.select_rgbd_frames(kf)
    B.upload_rgbd_frames(bgr[kf], sensor_ref.resize_depth(depth[kf], dcam, ccam))
    assert A.use_rgbd_level(1) == B.use_rgbd_level(1) == (ccam[0] // 2, ccam[1] // 2)
    shell = 2.0 * float(s["voxel_size"])
    for e in (A, B):
        e.set_camera(np.ascontiguousarray(s["poses"][kf]), np.array(ccam[2:], np.float64), np.zeros(5))
    le = engine.default_lighting_params()
    le.thres_shell, le.subvolume_size = shell, 0.04
    la, lb = A.estimate_lighting(le), B.estimate_lighting(le)
    assert la.usable and (la.num_subvolumes, la.num_data_rows, la.lm_iterations) == (lb.num_subvolumes, lb.num_data_rows, lb.lm_iterations)
    sha, shb = A.download_lighting()[1], B.download_lighting()[1]
    assert np.abs(sha - shb).max() <= 1e-8 * np.abs(sha).max()
    # the estimate sums with double atomics, so two engines can differ in the last bits (DESIGN.md §6k): both iterate on A's SH
    sh = A.download_voxel_sh()[0]
    for e in (A, B):
        e.set_sh(sh)
    gp = default_params()
    gp.thres_shell = shell
    gp.forced_cg_iterations = 4
    ia, ib = A.gn_iteration(gp), B.gn_iteration(gp)
    assert ia.type_residuals[0] > 0 and _info_bytes(ia) == _info_bytes(ib)
    xa, xb = A.download_state(), B.download_state()
    for k in xa:
        assert xa[k].tobytes() == xb[k].tobytes(), k
    assert A.download_colors().tobytes() == B.download_colors().tobytes()


def test_refusals_leave_both_stores_and_the_engine_usable():
    from intrinsic3d_b200 import engine
    s, dcam, depth, cams = _cams()
    ccam = cams["color_x2"]
    bgr = _bgr(len(depth), ccam, seed=6)
    inp = (dcam, depth, ccam, bgr) + _inputs(s)[4:]
    e = _engine()
    L = e.L

    def p(a, t):
        return a.ctypes.data_as(C.POINTER(t))
    sc = np.zeros(8)
    ids = np.array([0, 1], np.int32)
    pose = np.zeros((2, 12), np.float32)

    def refused(rc, word):
        assert rc != 0
        assert word in L.i3d_last_error(e.h).decode(), L.i3d_last_error(e.h).decode()

    dc, cc = engine.fusion_camera(dcam), engine.fusion_camera(ccam)
    refused(L.i3d_sensor_keyframe_scores(e.h, p(sc, C.c_double)), "no frames in the sensor store")
    refused(L.i3d_select_rgbd_frames(e.h, 2, p(ids, C.c_int32)), "no frames in the sensor store")
    refused(L.i3d_sensor_frames_add(e.h, 1, p(depth, C.c_float), p(bgr, C.c_uint8)), "no sensor store")
    refused(L.i3d_fusion_integrate_sensor(e.h, 2, p(ids, C.c_int32), p(pose, C.c_float), p(pose, C.c_float)), "no fusion in progress")
    # the first frame store, filled from the host, must survive everything below
    kb, kd = _bgr(2, (12, 10), seed=7), np.random.default_rng(8).random((2, 10, 12)).astype(np.float32)
    e.upload_rgbd_frames(kb, kd)

    def first_store_intact():
        assert e.use_rgbd_level(0) == (12, 10)
        lg, dg, cg = e.debug_frames(with_color=True)
        assert cg.tobytes() == kb.tobytes() and dg.tobytes() == kd.tobytes()

    for bad in (engine.fusion_camera((0, 120, 100.0, 100.0, 80.0, 60.0)), engine.fusion_camera((160, 120, 0.0, 100.0, 80.0, 60.0)),
                engine.fusion_camera((160, 120, 100.0, float("nan"), 80.0, 60.0))):
        refused(L.i3d_sensor_frames_begin(e.h, C.byref(bad), C.byref(cc), 3), "bad camera")
        refused(L.i3d_sensor_frames_begin(e.h, C.byref(dc), C.byref(bad), 3), "bad camera")
    refused(L.i3d_sensor_frames_begin(e.h, C.byref(dc), C.byref(cc), 0), "capacity")
    assert e.sensor_num_frames() == 0
    first_store_intact()

    e.sensor_frames_begin(dcam, ccam, 3)
    e.sensor_frames_add(depth[:2], bgr[:2])
    first_store_intact()                                          # the sensor store is independent of it
    scores = e.sensor_keyframe_scores()

    def sensor_intact():
        assert e.sensor_num_frames() == 2
        assert e.sensor_keyframe_scores().tobytes() == scores.tobytes()

    refused(L.i3d_sensor_frames_add(e.h, 2, p(depth, C.c_float), p(bgr, C.c_uint8)), "capacity")
    refused(L.i3d_sensor_frames_add(e.h, 0, p(depth, C.c_float), p(bgr, C.c_uint8)), "F > 0")
    sensor_intact()
    first_store_intact()
    for bad_ids, n, word in ((ids, 0, "n > 0"), (np.array([0, 2], np.int32), 2, "out of range"), (np.array([-1], np.int32), 1, "out of range")):
        refused(L.i3d_select_rgbd_frames(e.h, n, p(bad_ids, C.c_int32)), word)
        sensor_intact()
        first_store_intact()
    bad = engine.fusion_camera((160, 120, -1.0, 100.0, 80.0, 60.0))
    refused(L.i3d_sensor_frames_begin(e.h, C.byref(bad), C.byref(cc), 3), "bad camera")
    sensor_intact()

    # a refused store fusion keeps the fusion in progress; the following valid call fuses as the host path does
    fp = _params(s)
    e.fusion_begin(fp)
    refused(L.i3d_fusion_integrate_sensor(e.h, 2, p(np.array([0, 5], np.int32), C.c_int32), p(pose, C.c_float), p(pose, C.c_float)), "out of range")
    refused(L.i3d_fusion_integrate_sensor(e.h, 0, p(ids, C.c_int32), p(pose, C.c_float), p(pose, C.c_float)), "n > 0")
    sensor_intact()
    e.fusion_integrate_sensor([1, 0], inp[4][[1, 0]], inp[5][[1, 0]])
    _same(e.fusion_volume(), _fuse_host(fp, inp, [1, 0]).fusion_volume())
    e.fusion_finish()
    e.select_rgbd_frames([1])
    assert e.use_rgbd_level(0) == (ccam[0], ccam[1])
    assert e.debug_frames()[1].tobytes() == sensor_ref.resize_depth(depth[1:2], dcam, ccam).tobytes()
    sensor_intact()
