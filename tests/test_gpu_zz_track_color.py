"""GPU tests of tracking with colour as well as depth (the _rgbd calls, DESIGN.md §6p): planes byte-equal and sums to 1e-12 against the
restatement tests/track_color_ref.py, the depth-only bytes at weight 0, byte identity across batches, passes and chunked calls, the identity
with fusion_finish + track_sensor_frames_rgbd, the golden fixture, the refusals and the state a call leaves alone, and the C2 odometry and
finished-grid accuracy."""
import ctypes as C
import os

import numpy as np
import pytest

import track_color_ref as tc
import track_ref as tr
from test_gpu_zz_odometry import _engine, _volume_bytes
from test_gpu_zz_track import _rel
from test_odometry import ANCHORED, dense_tiny, live_grid

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _fused(s, k):
    """an engine with the scene's first k frames fused at their true poses (fusion still in progress)"""
    e, c2w, w2c = _engine(s)
    e.fusion_integrate_sensor(np.arange(k), c2w[:k], w2c[:k])
    return e


def _check_against_restatement(e, s, ids, start, levels, iterations):
    from fusion_ref import scene_inputs
    dcam, depth, ccam, bgr, _, _ = scene_inputs(s)
    v = e.fusion_volume()
    keep = v["weight"] > 0
    grid = live_grid(v, np.float32(s["voxel_size"]))
    inten = {f: tc.frame_intensity(bgr[f], ccam, dcam) for f in ids}
    out = e.fusion_track_sensor_frames_rgbd(ids, start, num_levels=levels, iterations=iterations)
    p = tr.params(num_levels=levels, iterations=iterations)
    c = tc.color_params()
    frames = [tc.ColorFrame(depth[f], inten[f], start[k], dcam, p, c, grid=grid, rgb=v["rgb"][keep]).run() for k, f in enumerate(ids)]
    n = len(ids)
    sums, T = e.debug_track_system(n)
    csum = e.debug_track_color_system(n)
    for k, f in enumerate(frames):
        info = out[1][k]
        assert [f.status, f.iterations, f.correspondences] == [info["status"], info["iterations"], info["correspondences"]], k
        assert f.sys[28] == sums[k, 28] and _rel(sums[k], f.sys), (k, sums[k], f.sys)
        assert f.sys_c[28] == csum[k, 28] and _rel(csum[k], f.sys_c), (k, csum[k], f.sys_c)
        assert [f.first[0], f.last[0]] == [info["color"]["first_rows"], info["color"]["last_rows"]]
        assert np.abs(np.array(f.w2c) - out[0][k]).max() <= 1e-12 and np.abs(np.array(f.T) - T[k]).max() <= 1e-12
    for l in range(levels):
        P = e.debug_track_color_planes(l, n)
        for k, f in enumerate(frames):
            assert P["intensity"][k].tobytes() == f.inten[l].tobytes(), ("intensity", l, k)
            assert P["grad_x"][k].tobytes() == f.grads[l][0].tobytes() and P["grad_y"][k].tobytes() == f.grads[l][1].tobytes(), (l, k)
            if l == 0:
                assert P["model_intensity"][k].tobytes() == f.pint.tobytes(), ("model_intensity", k)
    return out, frames


def test_planes_sums_and_poses_against_the_restatement():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e = _fused(s, 6)
    ids = [6, 8, 3]
    start = tr.perturb(true[ids], 1.0, 0.01, seed=2)
    _check_against_restatement(e, s, ids, start, 3, (0, 0, 0))          # the level-0 systems at the input pose
    out, frames = _check_against_restatement(e, s, ids, start, 3, (3, 2, 1))
    assert all(f.last[0] > 100 for f in frames)
    assert e.phase_ms("track_color") > 0 and e.phase_count("track_photo_correspondences") > 0


def test_weight_zero_gives_the_depth_only_bytes():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    zero = dict(weight=0.0)
    ids = [5, 7, 9]
    start = tr.perturb(true[ids], 1.0, 0.01, seed=3)
    e = _fused(s, 5)
    a = e.fusion_track_sensor_frames(ids, start)
    sa = e.debug_track_system(3)
    b = e.fusion_track_sensor_frames_rgbd(ids, start, color=zero)
    sb = e.debug_track_system(3)
    assert a[0].tobytes() == b[0].tobytes() and sa[0].tobytes() == sb[0].tobytes() and sa[1].tobytes() == sb[1].tobytes()
    assert a[1] == [{k: v for k, v in i.items() if k != "color"} for i in b[1]]
    e.fusion_finish()
    a = e.track_sensor_frames(ids, start, "fused")
    sa = e.debug_track_system(3)
    b = e.track_sensor_frames_rgbd(ids, start, "fused", color=zero)
    sb = e.debug_track_system(3)
    assert a[0].tobytes() == b[0].tobytes() and sa[0].tobytes() == sb[0].tobytes()
    assert a[1] == [{k: v for k, v in i.items() if k != "color"} for i in b[1]]
    e1, _, _ = _engine(s)
    e2, _, _ = _engine(s)
    a = e1.fusion_track_and_integrate_sensor(list(range(12)), true[0])
    b = e2.fusion_track_and_integrate_sensor_rgbd(list(range(12)), true[0], color=zero)
    assert a[0].tobytes() == b[0].tobytes() and _volume_bytes(e1) == _volume_bytes(e2)
    assert a[1] == [{k: v for k, v in i.items() if k != "color"} for i in b[1]]


def test_a_frame_does_not_depend_on_its_batch_or_pass():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e = _fused(s, 8)
    ids = list(range(8, 48))                                            # 40 frames: two passes of I3D_TRACK_CHUNK
    start = tr.perturb(true[ids], 1.0, 0.01, seed=4)
    full = e.fusion_track_sensor_frames_rgbd(ids, start)
    rev = e.fusion_track_sensor_frames_rgbd(ids[::-1], start[::-1])
    assert full[0].tobytes() == rev[0][::-1].tobytes() and full[1] == rev[1][::-1]
    for k in (0, 31, 32, 39):
        one = e.fusion_track_sensor_frames_rgbd([ids[k]], start[k:k + 1])
        assert one[0][0].tobytes() == full[0][k].tobytes() and one[1][0] == full[1][k], k


def _run(s, ids, first, chunks):
    e, _, _ = _engine(s)
    outs = []
    for c, part in enumerate(np.array_split(np.asarray(ids, np.int32), chunks)):
        outs.append(e.fusion_track_and_integrate_sensor_rgbd(part, first if c == 0 else None))
    return np.concatenate([o[0] for o in outs]).tobytes() + repr([i for o in outs for i in o[1]]).encode(), _volume_bytes(e)


def test_loop_bytes_across_calls():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    ids = [k % 72 for k in range(80)]
    assert _run(s, ids, true[0], 1) == _run(s, ids, true[0], 4)


@pytest.mark.parametrize("skip", [True, False])
def test_identity_with_finish_and_track(skip):
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    for k in (1, 4):
        e = _fused(s, k)
        e.set_render_skip(skip)
        ids = [k, k + 1, k + 2]
        start = tr.perturb(true[ids], 1.0, 0.005, seed=k)
        vol = _volume_bytes(e)
        live = e.fusion_track_sensor_frames_rgbd(ids, start)
        live_sys, live_c = e.debug_track_system(3), e.debug_track_color_system(3)
        live_planes = [e.debug_track_color_planes(l, 3) for l in range(3)]
        assert _volume_bytes(e) == vol
        e.fusion_finish()
        fin = e.track_sensor_frames_rgbd(ids, start, "fused")
        fin_sys, fin_c = e.debug_track_system(3), e.debug_track_color_system(3)
        fin_planes = [e.debug_track_color_planes(l, 3) for l in range(3)]
        assert live[0].tobytes() == fin[0].tobytes() and live[1] == fin[1], (k, skip)
        assert live_sys[0].tobytes() == fin_sys[0].tobytes() and live_c.tobytes() == fin_c.tobytes()
        for a, b in zip(live_planes, fin_planes):
            for name in a:
                assert a[name].tobytes() == b[name].tobytes(), (k, skip, name)


def test_golden_fixture_on_device():
    from intrinsic3d_b200.engine import Engine
    g = np.load(os.path.join(HERE, "golden", "tiny_track_color.npz"))
    e = Engine(0)
    sdf = g["sdf"].astype(np.float64)
    e.upload_grid(g["xyz"], sdf, sdf, np.zeros_like(sdf), g["weight"], g["rgb"], float(g["voxel_size"]))
    dcam = tuple(float(x) for x in g["dcam"])
    dcam = (int(dcam[0]), int(dcam[1])) + dcam[2:]
    e.sensor_frames_begin(dcam, dcam, len(g["depth"]))
    e.sensor_frames_add(np.ascontiguousarray(g["depth"]), np.ascontiguousarray(g["bgr"]))
    ids = g["ids"].tolist()
    out, info = e.track_sensor_frames_rgbd(ids, g["pose_in"], "fused", num_levels=int(g["num_levels"]), iterations=g["iterations"].tolist())
    sums, _ = e.debug_track_system(len(ids))
    csum = e.debug_track_color_system(len(ids))
    for k in range(len(ids)):
        assert [info[k]["status"], info[k]["iterations"], info[k]["correspondences"]] == g["outcome"][k].tolist()
        assert [info[k]["color"]["first_rows"], info[k]["color"]["last_rows"]] == g["color_rows"][k].tolist()
        assert _rel(sums[k], g["sums"][k]) and _rel(csum[k], g["color_sums"][k])
        assert np.abs(out[k] - g["pose_out"][k]).max() <= 1e-12
    P = e.debug_track_color_planes(0, len(ids))
    assert P["model_intensity"].tobytes() == g["model_intensity"].tobytes()
    assert P["intensity"].tobytes() == g["intensity_0"].tobytes() and P["grad_x"].tobytes() == g["grad_x_0"].tobytes()


def test_refusals_and_state_left_alone():
    from intrinsic3d_b200 import engine
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e = _fused(s, 3)
    vol = _volume_bytes(e)
    bad = [(dict(weight=-0.1), "weight"), (dict(weight=float("nan")), "weight"), (dict(max_color_diff=0.0), "max_color_diff"),
           (dict(max_color_diff=float("inf")), "max_color_diff"), (dict(min_color_gradient=-1.0), "min_color_gradient"),
           (dict(min_color_gradient=float("nan")), "min_color_gradient")]
    for color, text in bad:
        with pytest.raises(RuntimeError, match=text):
            e.fusion_track_sensor_frames_rgbd([3], true[3:4], color=color)
        with pytest.raises(RuntimeError, match=text):
            e.fusion_track_and_integrate_sensor_rgbd([3], true[3], color=color)
        assert _volume_bytes(e) == vol
    with pytest.raises(RuntimeError, match="num_levels"):
        e.fusion_track_sensor_frames_rgbd([3], true[3:4], num_levels=5)
    with pytest.raises(RuntimeError, match="no grid"):
        e.track_sensor_frames_rgbd([3], true[3:4])
    p, out, ids = engine.default_track_params(), np.empty((1, 12)), np.array([3], np.int32)
    pin = np.ascontiguousarray(true[3:4])
    assert e.L.i3d_fusion_track_sensor_frames_rgbd(e.h, 1, ids.ctypes.data_as(C.POINTER(C.c_int32)), pin.ctypes.data_as(C.POINTER(C.c_double)),
                                                   C.byref(p), None, out.ctypes.data_as(C.POINTER(C.c_double)), None, None) != 0
    assert b"color params" in e.L.i3d_last_error(e.h)
    assert _volume_bytes(e) == vol


def test_refinement_render_and_mesh_unchanged_by_rgbd_tracking(tiny_scene):
    """a GN iteration, i3d_download_render and the resident mesh are byte-identical with and without an _rgbd call in between"""
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.engine import Engine
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    F, H, W = s["depth"].shape
    dcam = (W, H) + tuple(float(v) for v in s["intr"])

    def run(track):
        e = Engine(0)
        e.load_scene(s)
        e.sensor_frames_begin(dcam, dcam, F)
        e.sensor_frames_add(s["depth"], make_color_frames(s))
        e.render_keyframes([0, 3])
        m = e.extract_mesh("refined")
        if track:
            e.track_sensor_frames_rgbd(list(range(F)), tr.aa_to_rt(s["poses"]), "refined")
        Wf, Hf = e.frame_size
        planes = [np.empty((2, Hf, Wf), np.float32), np.empty((2, Hf, Wf, 3), np.float32)] + [np.empty((2, Hf, Wf), np.float32) for _ in range(3)]
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


def _c2(frames):
    import torch
    from intrinsic3d_b200.scene import config_scene
    return config_scene("c2", device="cuda:0" if torch.cuda.is_available() else "cpu", frames=frames)


@pytest.mark.xfail(strict=True, reason="measured on an H100: the gates break at frame 35 with the default weight 0.05 (depth-only: frame "
                   "29; 0.1: frame 8; 0.2: frame 3); the fused voxel colours are a blurred, biased model of the frames (DESIGN.md §6p)")
def test_c2_odometry_all_200_frames_with_colour():
    """Headline: C2 geometry, 200 frames (2.5 deg of orbit per frame), frame 0 anchored at its true pose, default colour parameters.
    The depth-only loop holds only the first 25 frames (DESIGN.md §6o).  Not met: see the xfail reason."""
    s = _c2(200)
    true = tr.aa_to_rt(s["poses_true"])
    e, c2w, w2c = _engine(s)
    ids = np.arange(200, dtype=np.int32)
    out, info = e.fusion_track_and_integrate_sensor_rgbd(ids, true[0])
    st = [i["status"] for i in info]
    r, t = tr.pose_errors(out, true[ids])
    bad = [k for k in range(200) if st[k] not in (0, ANCHORED) or r[k] > 0.2 or t[k] > 0.002]
    print("C2 rgbd odometry, 200 frames: rot deg max %.4f median %.4f, centre mm max %.4f median %.4f, first failing frame %s" %
          (r.max(), np.median(r), 1e3 * t.max(), 1e3 * np.median(t), bad[:1]))
    if bad:
        k = bad[0]
        print("frame %d: status %d, rot %.4f deg, centre %.4f mm, info %s" % (k, st[k], r[k], 1e3 * t[k], info[k]))
    tracked = e.fusion_volume()
    ref, _, _ = _engine(s)
    ref.fusion_integrate_sensor(ids, c2w[ids], w2c[ids])
    fused = ref.fusion_volume()
    ka, kb = tracked["weight"] > 0, fused["weight"] > 0
    A = {tuple(x): i for i, x in enumerate(tracked["xyz"][ka])}
    common = [(A[tuple(x)], j) for j, x in enumerate(fused["xyz"][kb]) if tuple(x) in A]
    ia, ib = np.array([c[0] for c in common]), np.array([c[1] for c in common])
    dsdf = np.abs(tracked["sdf"][ka][ia].astype(np.float64) - fused["sdf"][kb][ib]) / float(s["voxel_size"])
    print("C2 grid, 200 frames: voxel overlap %.4f, median |dsdf| %.4f voxel" % (len(common) / max(ka.sum(), kb.sum()), np.median(dsdf)))
    assert st[0] == ANCHORED and not bad, bad[:5]
    assert np.median(dsdf) <= 0.1


@pytest.mark.xfail(strict=True, reason="measured on an H100 at the default weight 0.05: rotation up to 0.15 deg and camera centre up "
                   "to 0.98 mm against 0.011 deg / 0.09 mm depth-only; the photometric residual at the true pose is about 0.04 rms "
                   "(DESIGN.md §6p)")
def test_c2_finished_grid_track_no_worse_than_depth_only():
    """C2 fused from the store at the true poses, all 50 frames from a seeded 5 mm / 0.5 deg perturbation: §6n measured rotation at most
    0.011 deg and camera centre at most 0.09 mm depth-only."""
    s = _c2(50)
    true = tr.aa_to_rt(s["poses_true"])
    e, c2w, w2c = _engine(s)
    ids = np.arange(50, dtype=np.int32)
    e.fusion_integrate_sensor(ids, c2w, w2c)
    e.fusion_finish()
    start = tr.perturb(true, 0.5, 0.005, seed=7)
    out, info = e.track_sensor_frames_rgbd(ids, start, "fused")
    r, t = tr.pose_errors(out, true)
    print("C2 finished grid with colour: rot deg max %.4f median %.4f, centre mm max %.4f median %.4f" %
          (r.max(), np.median(r), 1e3 * t.max(), 1e3 * np.median(t)))
    assert all(i["status"] == 0 for i in info)
    assert r.max() <= 0.011 and t.max() <= 0.00009, (r.max(), t.max())
