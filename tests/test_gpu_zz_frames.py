"""GPU parity of the keyframe blur scores and the device RGB-D pyramid (i3d_keyframe_scores, i3d_upload_rgbd_frames, i3d_use_rgbd_level)
against the numpy float32 restatement in tests/frames_ref.py: planes byte-equal, scores within 1e-13 (the double plane sums are taken in
another fixed order), and a level built on the device drives the refinement exactly as the same planes uploaded from the host."""
import ctypes as C
import os

import numpy as np
import pytest

import frames_ref as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frames(F, W, H, seed=0, blur_every=3):
    """Seeded colour patterns with noise, every `blur_every`-th frame box-blurred; depth with holes."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    bgr = np.empty((F, H, W, 3), np.uint8)
    for f in range(F):
        ph = rng.uniform(0, 2 * np.pi, 3)
        for c in range(3):
            v = 128 + 70 * np.sin(xx / (5 + 2 * c + f % 4) + ph[c]) * np.cos(yy / (6 + c) - ph[c]) + rng.integers(-20, 21, (H, W))
            if blur_every and f % blur_every == 1:
                for ax in (0, 1):
                    v = sum(np.roll(v, s, axis=ax) for s in range(-2, 3)) / 5.0
            bgr[f, :, :, c] = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    depth = (0.8 + 0.5 * rng.random((F, H, W))).astype(np.float32)
    depth[rng.random((F, H, W)) < 0.25] = 0.0
    return bgr, depth


def _engine():
    from intrinsic3d_b200.engine import Engine
    return Engine(0)


# smallest accepted size for level 2: level 1 must keep 3 px on each axis, so level 0 needs 6
@pytest.mark.parametrize("W,H,F", [(640, 480, 3), (161, 121, 4), (6, 6, 2), (7, 6, 2)])
@pytest.mark.parametrize("given_lum", [False, True])
def test_levels_byte_equal(W, H, F, given_lum):
    bgr, depth = _frames(F, W, H, seed=W + H)
    lum = np.random.default_rng(5).random((F, H, W)).astype(np.float32) if given_lum else None
    L, D = R.pyramid(bgr, depth, 3, lum=lum)
    e = _engine()
    e.upload_rgbd_frames(bgr, depth, lum)
    for lvl in (2, 1, 0):
        assert e.use_rgbd_level(lvl) == (L[lvl].shape[2], L[lvl].shape[1])
        lg, dg, cg = e.debug_frames(with_color=(lvl == 0))
        assert lg.tobytes() == L[lvl].tobytes(), lvl
        assert dg.tobytes() == D[lvl].tobytes(), lvl
        if lvl == 0:
            assert cg.tobytes() == bgr.tobytes()


@pytest.mark.parametrize("W,H,F", [(640, 480, 6), (161, 121, 7), (5, 5, 3)])
def test_scores_match_restatement(W, H, F):
    bgr, _ = _frames(F, W, H, seed=2 * W)
    bgr[0] = 90                                            # constant frame: NaN, as in the reference
    ref = R.blur_scores(bgr)
    got = _engine().keyframe_scores(bgr)
    assert np.isnan(got[0]) and (np.isnan(got) == np.isnan(ref)).all()
    ok = ~np.isnan(ref)
    assert ok.sum() >= 1 and np.abs(got[ok] - ref[ok]).max() <= 1e-13, np.abs(got[ok] - ref[ok]).max()


def test_selection_matches_on_separated_scene():
    from intrinsic3d_b200.keyframes import select_keyframes
    bgr, _ = _frames(24, 161, 121, seed=9, blur_every=2)
    ref = R.blur_scores(bgr)
    got = _engine().keyframe_scores(bgr)
    for beg in range(0, 24, 5):                            # the leader of every window is ahead of the runner-up by more than the tolerance
        w = np.sort(ref[beg:beg + 5])
        assert len(w) < 2 or w[-1] - w[-2] > 1e-12
    assert (select_keyframes(got, 5) == select_keyframes(ref, 5)).all()
    assert select_keyframes(got, 5).sum() == 5


def test_scores_independent_of_chunking():
    from intrinsic3d_b200.engine import KEYFRAME_CHUNK
    F = KEYFRAME_CHUNK + 3
    bgr, _ = _frames(F, 96, 72, seed=4)
    e = _engine()
    a = e.keyframe_scores(bgr)
    assert e.phase_count("keyframe_chunks") == 2
    b = e.keyframe_scores(bgr)
    one = np.concatenate([e.keyframe_scores(bgr[f:f + 1]) for f in range(F)])
    assert a.tobytes() == b.tobytes() == one.tobytes()
    assert _engine().keyframe_scores(bgr[::-1]).tobytes() == a[::-1].tobytes()


def test_golden_fixture_on_device():
    g = np.load(os.path.join(ROOT, "tests", "golden", "tiny_frames.npz"))
    e = _engine()
    assert np.abs(e.keyframe_scores(g["bgr"]) - g["scores"]).max() <= 1e-13
    e.upload_rgbd_frames(g["bgr"], g["depth"])
    for lvl, (kl, kd) in ((2, ("lum2", "depth2")), (1, ("lum1", "depth1"))):
        e.use_rgbd_level(lvl)
        lg, dg, _ = e.debug_frames()
        assert lg.tobytes() == g[kl].tobytes() and dg.tobytes() == g[kd].tobytes()
    e.use_rgbd_level(0)
    assert e.debug_frames()[0].tobytes() == g["lum0"].tobytes()


# ---- the device level drives the refinement like a host upload of the same planes ------------------------------------------------
def _info_bytes(info):
    return bytes(info)[:type(info).time_add.offset]       # every I3DIterInfo field before the wall-clock timers


def _loaded_pair(s, col):
    """Two engines with the same grid, camera and SH: A reads its frames from the device store, B gets host uploads."""
    A, B = _engine(), _engine()
    for e in (A, B):
        e.upload_grid(s["xyz"], s["sdf0"], s["sdf_refined"], s["albedo"], s["weight"], s["rgb"], s["voxel_size"])
    A.upload_rgbd_frames(col, s["depth"], s["lum"])
    A.use_rgbd_level(0)
    B.upload_frames(s["lum"], s["depth"], 1.0)
    B.upload_color_frames(col)
    for e in (A, B):
        e.set_camera(s["poses"], s["intr"], s["dist"])
        e.set_sh(s["sh"])
    return A, B


def _params(s):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    return p


def _same_state(A, B):
    sa, sb = A.download_state(), B.download_state()
    for k in sa:
        assert sa[k].tobytes() == sb[k].tobytes(), k


@pytest.mark.parametrize("lvl", [0, 1])
def test_gn_iteration_after_level_switch_matches_host_upload(tiny_scene, lvl):
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    L, D = R.pyramid(col, s["depth"], 2, lum=s["lum"])
    A, B = _loaded_pair(s, col)
    A.use_rgbd_level(lvl)
    B.upload_frames(L[lvl], D[lvl], 2.0 ** -lvl)
    p = _params(s)
    ia, ib = A.gn_iteration(p), B.gn_iteration(p)
    assert _info_bytes(ia) == _info_bytes(ib)
    _same_state(A, B)


def test_recolor_and_camera_state_across_level_switches(tiny_scene):
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    L, D = R.pyramid(col, s["depth"], 2, lum=s["lum"])
    A, B = _loaded_pair(s, col)
    p = _params(s)
    for e in (A, B):
        e.recompute_colors(0.02, 5)
    assert A.download_colors().tobytes() == B.download_colors().tobytes()
    ia, ib = A.gn_iteration(p), B.gn_iteration(p)
    assert ia.step_accepted and _info_bytes(ia) == _info_bytes(ib)
    poses = A.download_state()["poses"]
    assert np.abs(poses - s["poses"]).max() > 0                     # the live camera moved (it may now sit in the second buffer)
    A.use_rgbd_level(1)                                             # same F: the live camera state stays
    B.upload_frames(L[1], D[1], 0.5)
    assert A.download_state()["poses"].tobytes() == poses.tobytes()
    _same_state(A, B)
    ia, ib = A.gn_iteration(p), B.gn_iteration(p)
    assert _info_bytes(ia) == _info_bytes(ib)
    A.use_rgbd_level(0)                                             # back to level 0: colours resident again
    B.upload_frames(s["lum"], s["depth"], 1.0)
    B.upload_color_frames(col)
    for e in (A, B):
        e.recompute_colors(0.02, 5)
    assert A.download_colors().tobytes() == B.download_colors().tobytes()
    _same_state(A, B)


def test_cpp_refine_builds_levels_on_device():
    """nv::Intrinsic3D::refine with keyframes that carry only level 0 (+ colour) and num_rgbd_levels = 2 gives the same result as the call
    whose keyframes carry both levels, level 1 being the restatement's planes of the same level-0 inputs."""
    from intrinsic3d_b200.scene import make_color_frames, make_scene
    s = make_scene(radius_vox=12.0, frames=6, width=160, height=120, voxel_size=0.008, band=3.0, seed=6)
    col = make_color_frames(s)
    L, D = R.pyramid(col, s["depth"], 2, lum=s["lum"])
    one, calls1 = _run_cpp_refine(s, col, [L[0]], [D[0]])
    two, calls2 = _run_cpp_refine(s, col, L, D)
    assert calls1 == calls2 == 3
    assert len(one["xyz"]) > 0
    for k in two:
        assert one[k].tobytes() == two[k].tobytes(), k


def _run_cpp_refine(s, col, lums, depths):
    Hh = C.CDLL(os.path.join(ROOT, "intrinsic3d_b200", "libi3d_host.so"))

    def ptr(a, t):
        return a.ctypes.data_as(C.POINTER(t))
    F = s["lum"].shape[0]
    keep = s["weight"] > 0
    n = int(keep.sum())
    xyz = np.ascontiguousarray(s["xyz"][keep], np.int32)
    sdf = np.ascontiguousarray(s["sdf0"][keep], np.float32)
    wgt = np.ascontiguousarray(s["weight"][keep], np.float32)
    rgb = np.ascontiguousarray(s["rgb"][keep], np.uint8)
    lums = [np.ascontiguousarray(x, np.float32) for x in lums]
    depths = [np.ascontiguousarray(x, np.float32) for x in depths]
    nl = len(lums)
    Wl = np.array([x.shape[2] for x in lums], np.int32)
    Hl = np.array([x.shape[1] for x in lums], np.int32)
    lum_ptrs = (C.POINTER(C.c_float) * nl)(*[ptr(x, C.c_float) for x in lums])
    dep_ptrs = (C.POINTER(C.c_float) * nl)(*[ptr(x, C.c_float) for x in depths])
    colc = np.ascontiguousarray(col, np.uint8)
    poses = np.ascontiguousarray(s["poses"], np.float64).copy()
    intr = np.ascontiguousarray(s["intr"], np.float64).copy()
    dist = np.zeros(5)
    # num_grid_levels 2, num_rgbd_levels 2, thin shell 2 -> 1, clear distant voxels, occlusion 0.02, K 5, subvolume 0.06, SH reg 10,
    # 2 iterations, 50 LM steps, lambdas g 0.2, r 80 -> 10, s 120 -> 10, a 0.1
    cfg = np.array([2, 2, 2.0, 1.0, 1, 0.02, 5, 0.06, 10.0, 2, 50, 0.2, 80.0, 10.0, 120.0, 10.0, 0.1], np.float64)
    cap = 8 * n
    out = dict(xyz=np.zeros((cap, 3), np.int32), sdf0=np.zeros(cap), sdf=np.zeros(cap), alb=np.zeros(cap), w=np.zeros(cap, np.float32),
               rgb=np.zeros((cap, 3), np.uint8))
    m, vso, calls = C.c_int64(0), C.c_float(0), C.c_int32(0)
    rc = Hh.i3dh_run_refine(C.c_int64(n), ptr(xyz, C.c_int32), ptr(sdf, C.c_float), ptr(wgt, C.c_float), ptr(rgb, C.c_uint8), C.c_float(float(s["voxel_size"])),
                            C.c_int32(F), C.c_int32(nl), ptr(Wl, C.c_int32), ptr(Hl, C.c_int32), lum_ptrs, dep_ptrs, ptr(colc, C.c_uint8), ptr(poses, C.c_double),
                            ptr(intr, C.c_double), ptr(dist, C.c_double), ptr(cfg, C.c_double), C.c_int64(cap), C.byref(m), ptr(out["xyz"], C.c_int32),
                            ptr(out["sdf0"], C.c_double), ptr(out["sdf"], C.c_double), ptr(out["alb"], C.c_double), ptr(out["w"], C.c_float),
                            ptr(out["rgb"], C.c_uint8), C.byref(vso), C.byref(calls))
    assert rc == 0
    M = int(m.value)
    res = {k: v[:M] for k, v in out.items()}
    res.update(voxel_size=np.float32(vso.value), poses=poses, intr=intr, dist=dist)
    return res, int(calls.value)


# ---- refused inputs ---------------------------------------------------------------------------------------------------------------
def test_bad_input_fails_with_message_and_engine_stays_usable():
    e = _engine()
    L = e.L
    bgr, depth = _frames(2, 12, 10, seed=1)
    ok = e.keyframe_scores(bgr)

    def refused(rc, word):
        assert rc != 0
        assert word in L.i3d_last_error(e.h).decode()
        assert e.keyframe_scores(bgr).tobytes() == ok.tobytes()      # a following valid call succeeds

    def p(a, t):
        return a.ctypes.data_as(C.POINTER(t))
    sc = np.zeros(2)
    refused(L.i3d_keyframe_scores(e.h, 0, 12, 10, p(bgr, C.c_uint8), p(sc, C.c_double)), "F > 0")
    refused(L.i3d_keyframe_scores(e.h, 2, 4, 10, p(bgr, C.c_uint8), p(sc, C.c_double)), "5 px")
    refused(L.i3d_keyframe_scores(e.h, 2, 12, 4, p(bgr, C.c_uint8), p(sc, C.c_double)), "5 px")
    refused(L.i3d_use_rgbd_level(e.h, 0, None, None), "no frame store")
    refused(L.i3d_debug_get_frames(e.h, None, None, None), "no frames")
    refused(L.i3d_upload_rgbd_frames(e.h, 0, 12, 10, p(bgr, C.c_uint8), p(depth, C.c_float), None), "bad dimensions")
    refused(L.i3d_upload_rgbd_frames(e.h, 2, 12, 10, None, p(depth, C.c_float), None), "NULL")
    e.upload_rgbd_frames(bgr, depth)
    refused(L.i3d_use_rgbd_level(e.h, -1, None, None), "negative level")
    assert e.use_rgbd_level(2) == (3, 2)                               # 12 x 10 -> 6 x 5 -> 3 x 2
    refused(L.i3d_use_rgbd_level(e.h, 3, None, None), "at least 3 px")
    refused(L.i3d_debug_get_frames(e.h, None, None, p(np.zeros(100, np.uint8), C.c_uint8)), "colour")
    assert e.use_rgbd_level(0) == (12, 10)
    lg, dg, cg = e.debug_frames(with_color=True)
    assert cg.tobytes() == bgr.tobytes() and dg.tobytes() == depth.tobytes()
