"""CPU tests of dense RGB-D odometry (i3d_fusion_track_and_integrate_sensor, DESIGN.md §6o) through its restatement, composed here from the
fusion oracle (tests/fusion_ref.py), the march (tests/render_ref.py) and the tracker (tests/track_ref.py): the constant-velocity guess,
the anchor frame, the no-integrate-on-failure rule, accuracy on a dense tiny sequence, and the golden fixture tests/golden/tiny_odometry.npz.

The live grid the prediction is marched from is the fusion volume's voxels with weight > 0, as a render_ref.Grid of their float sdf: the
device march reads exactly those cubes and values, inside the box of exactly those voxels."""
import functools
import os

import numpy as np

import render_ref as rr
import track_ref as tr
from fusion_ref import FusionOracle, depth_range, scene_inputs

HERE = os.path.dirname(os.path.abspath(__file__))
ANCHORED = 4


def pose_compose(A, B):
    """A . B of R row-major | t [12] poses in double: [R_A R_B | R_A t_B + t_A], every sum left to right"""
    out = [0.0] * 12
    for a in range(3):
        for c in range(3):
            out[3 * a + c] = (A[3 * a] * B[c] + A[3 * a + 1] * B[3 + c]) + A[3 * a + 2] * B[6 + c]
        out[9 + a] = ((A[3 * a] * B[9] + A[3 * a + 1] * B[10]) + A[3 * a + 2] * B[11]) + A[9 + a]
    return out


def cv_guess(motion):
    """camera -> world guess from the motion state (1 or 2 poses, oldest first): T(k-1) . (T(k-2)^-1 . T(k-1)), or T(k-1)"""
    if len(motion) == 1:
        return list(motion[-1])
    prev, last = motion
    return pose_compose(last, pose_compose(tr.inverse(prev), last))


def live_grid(volume, voxel_size):
    """the fusion volume's voxels with weight > 0 as the march reads them, or None when there is none"""
    keep = volume["weight"] > 0
    if not keep.any():
        return None
    sdf = volume["sdf"][keep].astype(np.float64)
    return rr.Grid(volume["xyz"][keep], sdf, np.zeros_like(sdf), volume["weight"][keep], voxel_size)


class Odometry:
    """The loop restated: per frame the guess, then the anchor (empty volume) or the tracking of that frame from the guess against the
    live grid, and the integration at status 0 only."""

    def __init__(self, s, fusion_params=None, **track):
        self.dcam, self.depth, self.ccam, self.bgr, _, _ = scene_inputs(s)
        fp = dict(voxel_size=float(s["voxel_size"]), depth_min=depth_range(s)[0], depth_max=depth_range(s)[1])
        fp.update(fusion_params or {})
        self.vs = np.float32(fp["voxel_size"])
        self.fo = FusionOracle(**fp)
        self.p = tr.params(**track)
        self.motion = []
        self.frames = []            # per frame: (status, w2c out, the tracked Frame or None)

    def volume(self):
        return self.fo.volume()

    def step(self, fid, pose_first=None, motion=None):
        """one frame; pose_first (world -> camera) resets the motion state, `motion` (camera -> world poses) replaces it"""
        if motion is not None:
            self.motion = [list(m) for m in motion]
        if pose_first is not None:
            self.motion = []
            W = [float(a) for a in pose_first]
            T = tr.inverse(W)
        else:
            T = cv_guess(self.motion)
            W = tr.inverse(T)
        g = live_grid(self.volume(), self.vs)
        frame = None
        if g is None:
            status, Ti, Wi = ANCHORED, T, W
        else:
            frame = tr.Frame(self.depth[fid], np.array(W), self.dcam, self.p, grid=g).run()
            status = frame.status
            Ti, Wi = (frame.T, frame.w2c) if status == 0 else (None, None)
        if Ti is not None:
            self.fo.integrate(self.dcam, self.depth[fid:fid + 1], self.ccam, self.bgr[fid:fid + 1], np.array(Ti, np.float32)[None],
                              np.array(Wi, np.float32)[None])
            self.motion = (self.motion + [list(Ti)])[-2:]
        else:
            self.motion = [self.motion[-1] if self.motion else list(T)]
        out = Wi if Wi is not None else W
        self.frames.append((status, np.array(out), frame))
        return status, np.array(out), frame


@functools.lru_cache(maxsize=2)
def dense_tiny(frames=72):
    """the tiny scene with 5 degrees of orbit per frame"""
    from intrinsic3d_b200.scene import config_scene
    return config_scene("tiny", frames=frames)


def test_constant_velocity_guess_is_exact_on_a_constant_velocity_trajectory():
    rng = np.random.default_rng(3)
    from intrinsic3d_b200.scene import aa_to_rotation
    step_R = aa_to_rotation(np.array([0.01, -0.02, 0.015]))
    step_t = np.array([0.003, -0.001, 0.002])
    T0 = np.eye(4); T0[:3, :3] = aa_to_rotation(rng.normal(size=3) * 0.3); T0[:3, 3] = rng.normal(size=3)
    D = np.eye(4); D[:3, :3] = step_R; D[:3, 3] = step_t
    traj = [T0, T0 @ D, T0 @ D @ D]
    rt = [np.concatenate([m[:3, :3].reshape(-1), m[:3, 3]]).tolist() for m in traj]
    g = cv_guess(rt[:2])
    assert np.abs(np.array(g) - rt[2]).max() < 1e-12
    assert cv_guess(rt[1:2]) == rt[1]                                 # one previous pose: that pose


def test_anchor_frame_then_tracked_frames():
    s = dense_tiny(72)
    odo = Odometry(s, iterations=(4, 2, 2))
    true = tr.aa_to_rt(s["poses_true"])
    status, w2c, frame = odo.step(0, pose_first=true[0])
    assert status == ANCHORED and frame is None and np.array_equal(w2c, true[0])
    assert (odo.volume()["weight"] > 0).sum() > 1000
    st, w1, f1 = odo.step(1)
    assert st == 0 and f1 is not None
    assert np.abs(f1.pose_in - true[0]).max() < 1e-15                 # one previous pose: the guess is the anchor pose (inverted twice)
    r, t = tr.pose_errors(w1[None], true[1:2])
    assert r[0] < 0.5 and t[0] < 0.002, (r, t)


def test_failed_frame_is_not_integrated_and_resets_the_velocity():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    odo = Odometry(s, iterations=(2, 1, 1))
    odo.step(0, pose_first=true[0])
    odo.step(1)
    before = odo.volume()
    last = list(odo.motion[-1])
    odo.p = tr.params(iterations=(2, 1, 1), min_correspondences=10 ** 9)      # every system is too small: status 1
    st, w, f = odo.step(2)
    assert st == 1
    guess = tr.inverse(cv_guess([tr.inverse(true[0]), last]))
    assert np.array_equal(w, np.array(guess))                           # pose_out is the guess
    after = odo.volume()
    assert all(np.array_equal(before[k], after[k]) for k in before)     # not integrated
    assert odo.motion == [last]                                         # zero velocity at the last integrated pose


def run_sequence(s, ids, pose_first, **track):
    odo = Odometry(s, **track)
    for k, f in enumerate(ids):
        odo.step(f, pose_first=pose_first if k == 0 else None)
    return odo


def test_dense_tiny_sequence_tracks_every_frame():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    ids = list(range(12))
    odo = run_sequence(s, ids, true[0])
    st = [f[0] for f in odo.frames]
    assert st[0] == ANCHORED and all(x == 0 for x in st[1:]), st
    est = np.array([f[1] for f in odo.frames])
    r, t = tr.pose_errors(est, true[ids])
    print("tiny odometry: rot deg max", r.max(), "centre mm max", 1e3 * t.max())
    # the tiny sphere (radius 10 voxels) constrains a rotation about its centre only by its bumps: the rotation drifts by about 0.1 deg
    # per frame (measured: 0.99 deg after 11 tracked frames), the camera centre much less
    assert r.max() < 1.5 and t.max() < 0.005, (r, t)


def test_golden_fixture():
    g = np.load(os.path.join(HERE, "golden", "tiny_odometry.npz"))
    s = dense_tiny(int(g["frames"]))
    odo = run_sequence(s, g["ids"].tolist(), g["pose_first"], iterations=tuple(g["iterations"].tolist()))
    assert [f[0] for f in odo.frames] == g["status"].tolist()
    assert np.abs(np.array([f[1] for f in odo.frames]) - g["pose_out"]).max() <= 1e-12
    v = odo.volume()
    for k in ("xyz", "sdf", "weight", "rgb"):
        assert v[k].tobytes() == g[f"volume_{k}"].tobytes(), k
