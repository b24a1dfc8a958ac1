"""numpy restatement of the locally normalised intensity of the _ref calls (k_track_local_norm, intrinsic3d_b200/csrc/i3d_track.cuh,
DESIGN.md §6r) and of the _ref calls and the _ref odometry loop with it.

Built on tests/track_reference_ref.py (the reference model, its calls and its loop), tests/track_color_ref.py (the intensity pyramid,
gradients and photometric rows) and tests/track_ref.py, which it leaves as they are.  Every float operation is one numpy float32 operation
in the device's order, so the normalised planes, and the gradients and model planes read from them, are byte-equal.
"""
from __future__ import annotations

import numpy as np

import track_color_ref as tc
import track_ref as tr
import track_reference_ref as trr
from test_odometry import ANCHORED, cv_guess, live_grid

f32 = np.float32
# i3d_default_track_color_lni_params
DEFAULTS = dict(weight=0.005, max_color_diff=1.0, min_color_gradient=0.05, norm_radius=3, norm_eps=0.01)


def color_params(**over):
    """track_color_ref.color_params with the LNI defaults; norm_radius int, norm_eps float32"""
    c = tc.color_params(**dict(DEFAULTS, **over))
    c["norm_radius"] = int(c["norm_radius"])
    c["norm_eps"] = f32(c["norm_eps"])
    return c


def _clipped(P, r, op, init, axis):
    """op over the taps -r..r of every pixel along `axis`, clipped to the plane, in ascending order from init"""
    n = P.shape[axis]
    idx = np.arange(n)
    acc = np.full(P.shape, init, f32)
    for d in range(-r, r + 1):
        j = idx + d
        ok = (j >= 0) & (j < n)
        tap = np.take(P, np.clip(j, 0, n - 1), axis=axis)
        ok = ok[None, :] if axis == 1 else ok[:, None]
        acc = np.where(ok, op(acc, tap), acc)
    return acc


def local_norm(I, r, eps):
    """k_track_local_norm of one plane [H, W]: (I - mu) / sqrt(max(m2 - mu^2, 0) + eps^2) over the (2r+1)^2 window clipped to the plane,
    mu = S1 / n, m2 = S2 / n in float32 with the sums along the row first, then down the column of row sums, taps in ascending order;
    exactly 0 where the window's min equals its max"""
    I = np.asarray(I, f32)
    H, W = I.shape
    eps = f32(eps)
    planes = {}
    for name, P, op, init in (("s1", I, np.add, 0.0), ("s2", I * I, np.add, 0.0), ("lo", I, np.minimum, np.inf), ("hi", I, np.maximum, -np.inf)):
        planes[name] = _clipped(_clipped(P, r, op, f32(init), 1), r, op, f32(init), 0)
    x, y = np.arange(W), np.arange(H)
    nx = np.minimum(x + r, W - 1) - np.maximum(x - r, 0) + 1
    ny = np.minimum(y + r, H - 1) - np.maximum(y - r, 0) + 1
    n = (ny[:, None] * nx[None, :]).astype(f32)
    with np.errstate(all="ignore"):
        mu = planes["s1"] / n
        m2 = planes["s2"] / n
        var = np.maximum(m2 - mu * mu, f32(0.0))
        out = (I - mu) / np.sqrt(var + eps * eps)
    return np.where(planes["lo"] != planes["hi"], out, f32(0.0)).astype(f32)


def pyramid(inten0, levels, c):
    """the intensity pyramid the rows read: raw levels by pyrDown of the raw level above, each normalised when norm_radius > 0"""
    raw = tc.intensity_pyramid(inten0, levels)
    r = c.get("norm_radius", 0)
    return [local_norm(I, r, c["norm_eps"]) for I in raw] if r > 0 else raw


class LniFrame(trr.RefFrame):
    """track_reference_ref.RefFrame with both intensity pyramids through pyramid(): the model planes are sampled from the normalised
    reference, and the gradients and residuals read the normalised frame."""

    def __init__(self, depth0, inten0, pose_in, dcam, p, c, ref_depth0, ref_inten0, ref_pose, grid=None, prediction=None):
        L = p["num_levels"]
        cams = tr.level_cams(dcam, L)
        initial = None
        if prediction is None:
            rt_in = np.asarray(pose_in, np.float64).astype(f32)
            pdepth, pnrm, initial = tr.predict(grid, rt_in, cams[0], np.asarray(depth0, f32))
            prediction = (pdepth, pnrm)
        pdepth = np.asarray(prediction[0], f32)
        self.ref_pose = np.asarray(ref_pose, np.float64)
        self.ref_inten = pyramid(ref_inten0, L, c)
        self.ref_depth = tr.pyramid(ref_depth0, L)
        rt_in = np.asarray(pose_in, np.float64).astype(f32)
        rrt = self.ref_pose.astype(f32)
        self.models = [trr.ref_model(rt_in, cams[0], cams[l], l, pdepth, rrt, self.ref_inten[l], self.ref_depth[l], p["max_distance"])
                       for l in range(L)]
        H0, W0 = pdepth.shape
        self.pints = [trr.level0_layout(m, l, H0, W0) for l, m in enumerate(self.models)]
        tc.ColorFrame.__init__(self, depth0, inten0, pose_in, dcam, p, c, prediction=(prediction[0], prediction[1], self.pints[0]))
        self.inten = pyramid(inten0, L, c)
        self.grads = [tc.gradients(I) for I in self.inten]
        self.initial = initial


def track(grid, depth_frames, inten_frames, ids, pose_in, ref_ids, ref_pose, dcam, color=None, **over):
    """i3d_track_sensor_frames_rgbd_ref with color=dict(norm_radius=..., ...) restated: one LniFrame per id (run), in call order."""
    p = tr.params(**over)
    c = color_params(**(color or {}))
    return [LniFrame(depth_frames[f], inten_frames[f], pose_in[k], dcam, p, c, depth_frames[ref_ids[k]], inten_frames[ref_ids[k]], ref_pose[k],
                     grid=grid).run() for k, f in enumerate(ids)]


class LniOdometry(trr.RefOdometry):
    """The _ref loop with LNI restated: track_reference_ref.RefOdometry with LniFrame in place of RefFrame."""

    def __init__(self, s, fusion_params=None, color=None, **track):
        super().__init__(s, fusion_params, **track)
        self.c = color_params(**(color or {}))

    def step(self, fid, pose_first=None):
        """one frame; pose_first (world -> camera) resets the motion state and the reference"""
        if pose_first is not None:
            self.motion, self.ref = [], None
            W = [float(a) for a in pose_first]
            T = tr.inverse(W)
        else:
            T = cv_guess(self.motion)
            W = tr.inverse(T)
        g = live_grid(self.volume(), self.vs)
        frame, cinfo = None, (0, 0.0, 0, 0.0)
        if g is None:
            status, Ti, Wi = ANCHORED, T, W
        else:
            if self.ref is None:
                frame = tr.Frame(self.depth[fid], np.array(W), self.dcam, self.p, grid=g).run()
            else:
                rid, rT = self.ref
                frame = LniFrame(self.depth[fid], self.intensity(fid), np.array(W), self.dcam, self.p, self.c, self.depth[rid], self.intensity(rid),
                                 np.array(tr.inverse(rT)), grid=g).run()
                cinfo = (frame.first[0], frame.first[1], frame.last[0], frame.last[1])
            status = frame.status
            Ti, Wi = (frame.T, frame.w2c) if status == 0 else (None, None)
        if Ti is not None:
            self.fo.integrate(self.dcam, self.depth[fid:fid + 1], self.ccam, self.bgr[fid:fid + 1], np.array(Ti, np.float32)[None],
                              np.array(Wi, np.float32)[None])
            self.motion = (self.motion + [list(Ti)])[-2:]
            self.ref = (fid, list(Ti))
        else:
            self.motion = [self.motion[-1] if self.motion else list(T)]
        out = Wi if Wi is not None else W
        self.frames.append((status, np.array(out), frame))
        self.color_info.append(cinfo)
        return status, np.array(out), frame


def run_sequence(s, ids, pose_first, color=None, **track):
    odo = LniOdometry(s, color=color, **track)
    for k, f in enumerate(ids):
        odo.step(f, pose_first=pose_first if k == 0 else None)
    return odo
