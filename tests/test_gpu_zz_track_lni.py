"""GPU tests of the locally normalised intensity of the _ref calls (norm_radius > 0, DESIGN.md §6r): the frame's and the reference's
normalised planes, the gradients and the model planes byte-equal to the restatement tests/track_lni_ref.py at every level, sums and poses
to 1e-12, the loop frame by frame, the golden fixture, the _ref bytes at radius 0, byte identity across batches, passes and chunked calls,
the identity with fusion_finish + track_sensor_frames_rgbd_ref, the refusals and the state a call leaves alone, and the C2 accuracy."""
import ctypes as C
import os

import numpy as np
import pytest

import track_color_ref as tc
import track_lni_ref as tl
import track_ref as tr
from test_gpu_zz_odometry import _engine, _volume_bytes
from test_gpu_zz_track import _rel
from test_gpu_zz_track_color import _c2, _fused
from test_odometry import ANCHORED, dense_tiny, live_grid

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LNI = dict(norm_radius=5, norm_eps=0.01)


def _neighbours(ids):
    """each frame referenced to the frame before it (the first to the one after)"""
    return [ids[k - 1] if k > 0 else ids[1] for k in range(len(ids))]


def _check_planes(e, frames, levels):
    n = len(frames)
    for l in range(levels):
        P = e.debug_track_reference_planes(l, n)
        Q = e.debug_track_color_planes(l, n, model_intensity=False)
        for k, f in enumerate(frames):
            assert P["model"][k].tobytes() == f.models[l].tobytes(), ("model", l, k)
            assert P["ref_intensity"][k].tobytes() == f.ref_inten[l].tobytes(), ("ref_intensity", l, k)
            assert P["ref_depth"][k].tobytes() == f.ref_depth[l].tobytes(), ("ref_depth", l, k)
            assert Q["intensity"][k].tobytes() == f.inten[l].tobytes(), ("intensity", l, k)
            assert Q["grad_x"][k].tobytes() == f.grads[l][0].tobytes() and Q["grad_y"][k].tobytes() == f.grads[l][1].tobytes(), ("grad", l, k)


def _check_against_restatement(e, s, ids, start, refs, ref_pose, levels, iterations, color):
    from fusion_ref import scene_inputs
    dcam, depth, ccam, bgr, _, _ = scene_inputs(s)
    grid = live_grid(e.fusion_volume(), np.float32(s["voxel_size"]))
    inten = {f: tc.frame_intensity(bgr[f], ccam, dcam) for f in set(ids) | set(refs)}
    out = e.fusion_track_sensor_frames_rgbd_ref(ids, start, refs, ref_pose, color=color, num_levels=levels, iterations=iterations)
    p, c = tr.params(num_levels=levels, iterations=iterations), tl.color_params(**color)
    frames = [tl.LniFrame(depth[f], inten[f], start[k], dcam, p, c, depth[refs[k]], inten[refs[k]], ref_pose[k], grid=grid).run()
              for k, f in enumerate(ids)]
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
    _check_planes(e, frames, levels)
    return out, frames


@pytest.mark.parametrize("color", [LNI, dict(norm_radius=1, norm_eps=0.05), dict(norm_radius=8, norm_eps=0.002)])
def test_planes_sums_and_poses_against_the_restatement(color):
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e = _fused(s, 6)
    ids, refs = [6, 8, 3], [5, 8, 2]                                    # frame 8 is its own reference
    start = tr.perturb(true[ids], 1.0, 0.01, seed=2)
    ref_pose = true[refs]
    _check_against_restatement(e, s, ids, start, refs, ref_pose, 3, (0, 0, 0), color)
    out, frames = _check_against_restatement(e, s, ids, start, refs, ref_pose, 3, (3, 2, 1), color)
    assert all(f.last[0] > 100 for f in frames)
    assert all(np.isnan(f.models[l]).any() and np.isfinite(f.models[l]).any() for f in frames for l in range(3))
    assert all((f.inten[l] == 0).any() and (f.inten[l] != 0).any() for f in frames for l in range(3))     # constant windows give 0
    assert e.phase_ms("track_reference") > 0 and e.phase_count("track_photo_correspondences") > 0


def test_loop_frame_by_frame_against_the_restatement():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e, _, _ = _engine(s)
    odo = tl.LniOdometry(s, color=LNI)
    for k in range(6):
        first = true[0] if k == 0 else None
        out, info = e.fusion_track_and_integrate_sensor_rgbd_ref([k], first, color=LNI)
        st, w, f = odo.step(k, pose_first=first)
        assert info[0]["status"] == st and np.abs(out[0] - w).max() <= 1e-12, (k, info[0], st)
        c = info[0]["color"]
        assert (c["first_rows"], c["last_rows"]) == (odo.color_info[-1][0], odo.color_info[-1][2]), k
        v, r = e.fusion_volume(), odo.volume()
        assert all(v[n].tobytes() == r[n].tobytes() for n in ("xyz", "sdf", "weight", "rgb")), k
        if k >= 1:
            assert c["last_rows"] > 100
    assert odo.frames[0][0] == ANCHORED and odo.color_info[0] == (0, 0.0, 0, 0.0)


def test_golden_fixture_on_device():
    from intrinsic3d_b200.engine import Engine
    g = np.load(os.path.join(HERE, "golden", "tiny_track_lni.npz"))
    e = Engine(0)
    sdf = g["sdf"].astype(np.float64)
    e.upload_grid(g["xyz"], sdf, sdf, np.zeros_like(sdf), g["weight"], g["rgb"], float(g["voxel_size"]))
    dcam = tuple(float(x) for x in g["dcam"])
    dcam = (int(dcam[0]), int(dcam[1])) + dcam[2:]
    e.sensor_frames_begin(dcam, dcam, len(g["depth"]))
    e.sensor_frames_add(np.ascontiguousarray(g["depth"]), np.ascontiguousarray(g["bgr"]))
    ids = g["ids"].tolist()
    L = int(g["num_levels"])
    color = dict(norm_radius=int(g["norm_radius"]), norm_eps=float(g["norm_eps"]))
    out, info = e.track_sensor_frames_rgbd_ref(ids, g["pose_in"], g["ref_ids"], g["ref_pose"], "fused", color=color, num_levels=L,
                                               iterations=g["iterations"].tolist())
    sums, _ = e.debug_track_system(len(ids))
    csum = e.debug_track_color_system(len(ids))
    for k in range(len(ids)):
        assert [info[k]["status"], info[k]["iterations"], info[k]["correspondences"]] == g["outcome"][k].tolist()
        assert [info[k]["color"]["first_rows"], info[k]["color"]["last_rows"]] == g["color_rows"][k].tolist()
        assert _rel(sums[k], g["sums"][k]) and _rel(csum[k], g["color_sums"][k])
        assert np.abs(out[k] - g["pose_out"][k]).max() <= 1e-12
    for l in range(L):
        P = e.debug_track_reference_planes(l, len(ids))
        Q = e.debug_track_color_planes(l, len(ids), model_intensity=False)
        assert P["model"].tobytes() == g[f"model_{l}"].tobytes(), l
        assert P["ref_intensity"].tobytes() == g[f"ref_intensity_{l}"].tobytes() and Q["intensity"].tobytes() == g[f"intensity_{l}"].tobytes()


def test_radius_zero_gives_the_ref_bytes():
    """norm_radius 0 (whatever norm_eps) is the _ref call of DESIGN.md §6q, in all three calls"""
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    zero = dict(norm_radius=0, norm_eps=-3.0)
    ids = [5, 7, 9]
    start = tr.perturb(true[ids], 1.0, 0.01, seed=3)
    refs = _neighbours(ids)
    e = _fused(s, 5)
    for live in (True, False):
        fn = e.fusion_track_sensor_frames_rgbd_ref if live else (lambda *a, **k: e.track_sensor_frames_rgbd_ref(*a, "fused", **k))
        a = fn(ids, start, refs, true[refs])
        sa, ca = e.debug_track_system(3), e.debug_track_color_system(3)
        pa = [e.debug_track_reference_planes(l, 3) for l in range(3)]
        b = fn(ids, start, refs, true[refs], color=zero)
        sb, cb = e.debug_track_system(3), e.debug_track_color_system(3)
        pb = [e.debug_track_reference_planes(l, 3) for l in range(3)]
        assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1], live
        assert sa[0].tobytes() == sb[0].tobytes() and sa[1].tobytes() == sb[1].tobytes() and ca.tobytes() == cb.tobytes()
        assert all(x[k].tobytes() == y[k].tobytes() for x, y in zip(pa, pb) for k in x)
        if live:
            e.fusion_finish()
    e1, _, _ = _engine(s)
    e2, _, _ = _engine(s)
    a = e1.fusion_track_and_integrate_sensor_rgbd_ref(list(range(12)), true[0])
    b = e2.fusion_track_and_integrate_sensor_rgbd_ref(list(range(12)), true[0], color=zero)
    assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1] and _volume_bytes(e1) == _volume_bytes(e2)


def test_a_frame_does_not_depend_on_its_batch_or_pass():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e = _fused(s, 8)
    ids = list(range(8, 48))                                            # 40 frames: two passes of I3D_TRACK_CHUNK
    refs = _neighbours(ids)
    start = tr.perturb(true[ids], 1.0, 0.01, seed=4)
    rpose = true[refs]
    full = e.fusion_track_sensor_frames_rgbd_ref(ids, start, refs, rpose, color=LNI)
    rev = e.fusion_track_sensor_frames_rgbd_ref(ids[::-1], start[::-1], refs[::-1], rpose[::-1], color=LNI)
    assert full[0].tobytes() == rev[0][::-1].tobytes() and full[1] == rev[1][::-1]
    for k in (0, 31, 32, 39):
        one = e.fusion_track_sensor_frames_rgbd_ref([ids[k]], start[k:k + 1], [refs[k]], rpose[k:k + 1], color=LNI)
        assert one[0][0].tobytes() == full[0][k].tobytes() and one[1][0] == full[1][k], k


def _run(s, ids, first, chunks):
    e, _, _ = _engine(s)
    outs = []
    for c, part in enumerate(np.array_split(np.asarray(ids, np.int32), chunks)):
        outs.append(e.fusion_track_and_integrate_sensor_rgbd_ref(part, first if c == 0 else None, color=LNI))
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
        refs = [k - 1, k, k + 1]
        start = tr.perturb(true[ids], 1.0, 0.005, seed=k)
        vol = _volume_bytes(e)
        live = e.fusion_track_sensor_frames_rgbd_ref(ids, start, refs, true[refs], color=LNI)
        live_sys, live_c = e.debug_track_system(3), e.debug_track_color_system(3)
        live_planes = [e.debug_track_reference_planes(l, 3) for l in range(3)]
        assert _volume_bytes(e) == vol
        e.fusion_finish()
        fin = e.track_sensor_frames_rgbd_ref(ids, start, refs, true[refs], "fused", color=LNI)
        fin_sys, fin_c = e.debug_track_system(3), e.debug_track_color_system(3)
        fin_planes = [e.debug_track_reference_planes(l, 3) for l in range(3)]
        assert live[0].tobytes() == fin[0].tobytes() and live[1] == fin[1], (k, skip)
        assert live_sys[0].tobytes() == fin_sys[0].tobytes() and live_c.tobytes() == fin_c.tobytes()
        for a, b in zip(live_planes, fin_planes):
            for name in a:
                assert a[name].tobytes() == b[name].tobytes(), (k, skip, name)


def test_refusals_and_state_left_alone():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    e = _fused(s, 3)
    vol = _volume_bytes(e)
    e.fusion_track_sensor_frames_rgbd_ref([3], true[3:4], [2], true[2:3], color=LNI)
    planes = e.debug_track_reference_planes(0, 1)
    cases = [(dict(norm_radius=-1), "norm_radius"), (dict(norm_radius=9), "norm_radius"), (dict(norm_radius=2, norm_eps=0.0), "norm_eps"),
             (dict(norm_radius=2, norm_eps=-0.01), "norm_eps"), (dict(norm_radius=2, norm_eps=float("nan")), "norm_eps"),
             (dict(norm_radius=2, norm_eps=float("inf")), "norm_eps")]
    for color, text in cases:
        with pytest.raises(RuntimeError, match=text):
            e.fusion_track_sensor_frames_rgbd_ref([3], true[3:4], [2], true[2:3], color=color)
        with pytest.raises(RuntimeError, match=text):
            e.fusion_track_and_integrate_sensor_rgbd_ref([3], true[3], color=color)
        assert _volume_bytes(e) == vol
    # the voxel-model calls refuse any radius, even one the _ref calls take
    with pytest.raises(RuntimeError, match="voxel model"):
        e.fusion_track_sensor_frames_rgbd([3], true[3:4], color=dict(norm_radius=2, norm_eps=0.01))
    with pytest.raises(RuntimeError, match="voxel model"):
        e.fusion_track_and_integrate_sensor_rgbd([3], true[3], color=dict(norm_radius=2, norm_eps=0.01))
    assert _volume_bytes(e) == vol
    # nothing was tracked: the last call's planes are still there
    after = e.debug_track_reference_planes(0, 1)
    assert all(planes[k].tobytes() == after[k].tobytes() for k in planes)
    from intrinsic3d_b200 import engine
    p, cp, out = engine.default_track_params(), engine.default_track_color_params(), np.empty((1, 12))
    cp.norm_radius = 3
    cp.norm_eps = 0.01
    ids, pin = np.array([3], np.int32), np.ascontiguousarray(true[3:4])
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))                                  # noqa: E731
    ip = ids.ctypes.data_as(C.POINTER(C.c_int32))
    e.fusion_finish()
    assert e.L.i3d_track_sensor_frames_rgbd(e.h, 1, ip, dp(pin), C.byref(p), C.byref(cp), dp(out), None, None) != 0
    assert b"voxel model" in e.L.i3d_last_error(e.h)
    assert e.L.i3d_track_sensor_frames_rgbd_ref(e.h, 1, ip, dp(pin), ip, dp(pin), C.byref(p), C.byref(cp), dp(out), None, None) == 0


def test_refinement_render_and_mesh_unchanged_by_lni_tracking(tiny_scene):
    """a GN iteration, i3d_download_render and the resident mesh are byte-identical with and without an LNI _ref call in between"""
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
            poses = tr.aa_to_rt(s["poses"])
            refs = _neighbours(list(range(F)))
            e.track_sensor_frames_rgbd_ref(list(range(F)), poses, refs, poses[refs], "refined", color=LNI)
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


@pytest.mark.xfail(strict=True, reason="measured on an H100: every frame at status 0 but up to 0.035 deg and 0.25 mm at the "
                   "default LNI parameters (raw reference: 0.027 deg / 0.23 mm; depth only: 0.011 deg / 0.09 mm); the residual at the "
                   "true pose comes from resampling the unanti-aliased checker edges, which the normalisation does not remove "
                   "(DESIGN.md §6r)")
def test_c2_finished_grid_with_neighbour_references():
    """C2 fused from the store at the true poses, all 50 frames from the seeded 5 mm / 0.5 deg perturbation, each frame referenced to
    its neighbour (k - 1; frame 0 to frame 1) at its true pose, with the default LNI parameters: §6n's depth-only bounds, 0.011 deg and
    0.09 mm."""
    from intrinsic3d_b200.engine import default_track_color_lni_params
    s = _c2(50)
    true = tr.aa_to_rt(s["poses_true"])
    e, c2w, w2c = _engine(s)
    ids = np.arange(50, dtype=np.int32)
    e.fusion_integrate_sensor(ids, c2w, w2c)
    e.fusion_finish()
    start = tr.perturb(true, 0.5, 0.005, seed=7)
    refs = _neighbours(list(range(50)))
    color = dict(norm_radius=default_track_color_lni_params().norm_radius)
    out, info = e.track_sensor_frames_rgbd_ref(ids, start, refs, true[refs], "fused", color=color)
    r, t = tr.pose_errors(out, true)
    print("C2 finished grid, LNI reference model: rot deg max %.4f median %.4f, centre mm max %.4f median %.4f" %
          (r.max(), np.median(r), 1e3 * t.max(), 1e3 * np.median(t)))
    assert all(i["status"] == 0 for i in info)
    assert r.max() <= 0.011 and t.max() <= 0.00009, (r.max(), t.max())


@pytest.mark.xfail(strict=True, reason="measured on an H100: at the default LNI parameters the gates break at frame 37 (52 "
                   "frames at status 0; raw reference: frame 28, 56 frames; depth only: frame 29, 39 frames); grid median |dsdf| 0.56 "
                   "voxel; with clean colour frames (no modulation) the raw reference at 0.01 breaks at frame 28 as well, so appearance "
                   "compensation alone cannot reach the gate (DESIGN.md §6r)")
def test_c2_odometry_all_200_frames_with_lni():
    """Headline: C2 geometry, 200 frames, frame 0 anchored at its true pose, the _ref loop at the default LNI colour parameters: every
    other frame at status 0 within 0.2 deg and 2 mm, and the grid within a median |dsdf| of 0.1 voxel of the true-pose fusion."""
    from intrinsic3d_b200.engine import default_track_color_lni_params
    s = _c2(200)
    true = tr.aa_to_rt(s["poses_true"])
    e, c2w, w2c = _engine(s)
    ids = np.arange(200, dtype=np.int32)
    color = dict(norm_radius=default_track_color_lni_params().norm_radius)
    out, info = e.fusion_track_and_integrate_sensor_rgbd_ref(ids, true[0], color=color)
    st = [i["status"] for i in info]
    r, t = tr.pose_errors(out, true[ids])
    bad = [k for k in range(200) if st[k] not in (0, ANCHORED) or r[k] > 0.2 or t[k] > 0.002]
    print("C2 LNI odometry, 200 frames: status 0 %d, rot deg max %.4f median %.4f, centre mm max %.4f median %.4f, first failing "
          "frame %s" % (st.count(0), r.max(), np.median(r), 1e3 * t.max(), 1e3 * np.median(t), bad[:1]))
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
