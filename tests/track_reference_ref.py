"""numpy restatement of the reference model of the photometric term (k_track_ref_model, intrinsic3d_b200/csrc/i3d_track.cuh, DESIGN.md §6q)
and of the _ref calls and the _ref odometry loop built on it.

Built on tests/track_color_ref.py (the photometric rows and the combined system), tests/track_ref.py (the geometric term, the plain march
and the solve), tests/render_ref.py, tests/frames_ref.py / tests/sensor_ref.py (the intensity and depth pyramids) and test_odometry.Odometry
(the loop), which it leaves as they are.  Every float operation is one numpy float32 operation in the device's order, so the model,
reference intensity and reference depth planes are byte-equal, NaNs included.
"""
from __future__ import annotations

import numpy as np

import track_color_ref as tc
import track_ref as tr
from test_odometry import ANCHORED, Odometry, cv_guess, live_grid

f32 = np.float32
QNAN = np.array(0x7FC00000, np.uint32).view(f32)        # the kernel's "no model value"
REF_WEIGHT = 0.01                                       # i3d_default_track_color_ref_params


def color_params(**over):
    """track_color_ref.color_params with the _ref calls' default weight"""
    return tc.color_params(**dict(dict(weight=REF_WEIGHT), **over))


def ref_model(rt_in, cam0, cam, l, pdepth, ref_rt, ref_I, ref_D, max_distance):
    """k_track_ref_model of one frame at level l: the compact model plane [H_l, W_l] (QNAN where any test fails).  rt_in / ref_rt: the
    frame's input and the reference's world -> camera poses in float [12]; ref_I / ref_D: the reference's level-l intensity and depth."""
    H, W = ref_I.shape
    step = 1 << l
    vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    iu, iv = uu * step, vv * step
    zm = pdepth[iv, iu]
    ok = zm > 0
    R0 = np.asarray(rt_in, f32)
    Rr = np.asarray(ref_rt, f32)
    with np.errstate(all="ignore"):
        xn = (iu.astype(f32) - cam0["cx"]) / cam0["fx"]
        yn = (iv.astype(f32) - cam0["cy"]) / cam0["fy"]
        q = []
        for k in range(3):
            o = -((R0[k] * R0[9] + R0[3 + k] * R0[10]) + R0[6 + k] * R0[11])
            dr = (R0[k] * xn + R0[3 + k] * yn) + R0[6 + k]
            q.append(o + zm * dr)
        xr = tr.xform(Rr, Rr[9:], q)
        ok &= xr[2] > 0
        x = cam["fx"] * (xr[0] / xr[2]) + cam["cx"]
        y = cam["fy"] * (xr[1] / xr[2]) + cam["cy"]
        ok &= (x >= f32(1.0)) & (x < f32(W - 2)) & (y >= f32(1.0)) & (y < f32(H - 2))
        xs, ys = np.where(ok, x, f32(1.0)), np.where(ok, y, f32(1.0))
        d = ref_D[np.trunc(ys + f32(0.5)).astype(np.int64), np.trunc(xs + f32(0.5)).astype(np.int64)]
        ok &= (d > 0) & (np.abs(d - xr[2]) <= max_distance)
        xf, yf = np.floor(xs), np.floor(ys)
        val = tc._bilinear(np.asarray(ref_I, f32), xf.astype(np.int64), yf.astype(np.int64), xs - xf, ys - yf)
    return np.where(ok, val, QNAN).astype(f32)


def level0_layout(model, l, H0, W0):
    """the compact level-l model plane in the level-0 layout k_track_photo_rows reads (pixel (u, v) at (2^l v, 2^l u)); the rest QNAN"""
    out = np.full((H0, W0), QNAN, f32)
    H, W = model.shape
    s = 1 << l
    out[:H * s:s, :W * s:s] = model
    return out


class RefFrame(tc.ColorFrame):
    """One frame's joint problem with the reference model: the plain march at the input pose, the reference's intensity and depth
    pyramids by the frame's own rules, and per level the model plane of ref_model in place of the voxel model intensity."""

    def __init__(self, depth0, inten0, pose_in, dcam, p, c, ref_depth0, ref_inten0, ref_pose, grid=None, prediction=None):
        cams = tr.level_cams(dcam, p["num_levels"])
        initial = None
        if prediction is None:
            rt_in = np.asarray(pose_in, np.float64).astype(f32)
            pdepth, pnrm, initial = tr.predict(grid, rt_in, cams[0], np.asarray(depth0, f32))
            prediction = (pdepth, pnrm)
        pdepth = np.asarray(prediction[0], f32)
        self.ref_pose = np.asarray(ref_pose, np.float64)
        self.ref_inten = tc.intensity_pyramid(ref_inten0, p["num_levels"])
        self.ref_depth = tr.pyramid(ref_depth0, p["num_levels"])
        rt_in = np.asarray(pose_in, np.float64).astype(f32)
        rrt = self.ref_pose.astype(f32)
        self.models = [ref_model(rt_in, cams[0], cams[l], l, pdepth, rrt, self.ref_inten[l], self.ref_depth[l], p["max_distance"])
                       for l in range(p["num_levels"])]
        H0, W0 = pdepth.shape
        self.pints = [level0_layout(m, l, H0, W0) for l, m in enumerate(self.models)]
        super().__init__(depth0, inten0, pose_in, dcam, p, c, prediction=(prediction[0], prediction[1], self.pints[0]))
        self.initial = initial

    def photo_system(self, l):
        ok, J, r = tc.photo_rows(self.Tf(), self.rt_in, self.cams[0], self.cams[l], l, self.pdepth, self.pints[l], self.inten[l], *self.grads[l],
                                 self.depth[l], self.p["max_distance"], self.c)
        return tr.tile_sums(tr.values(J, r, ok))


def track(grid, depth_frames, inten_frames, ids, pose_in, ref_ids, ref_pose, dcam, color=None, **over):
    """i3d_track_sensor_frames_rgbd_ref restated: one RefFrame per id (run), in call order."""
    p = tr.params(**over)
    c = color_params(**(color or {}))
    return [RefFrame(depth_frames[f], inten_frames[f], pose_in[k], dcam, p, c, depth_frames[ref_ids[k]], inten_frames[ref_ids[k]], ref_pose[k],
                     grid=grid).run() for k, f in enumerate(ids)]


class RefOdometry(Odometry):
    """The _ref loop restated: test_odometry.Odometry with each tracked frame's model intensity from the last integrated frame at the
    camera -> world pose it was integrated with (world -> camera by track_ref.inverse); without one, depth alone and zero colour info."""

    def __init__(self, s, fusion_params=None, color=None, **track):
        super().__init__(s, fusion_params, **track)
        self.c = color_params(**(color or {}))
        self.inten = {}
        self.ref = None                 # (id, camera -> world)
        self.color_info = []

    def intensity(self, f):
        if f not in self.inten:
            self.inten[f] = tc.frame_intensity(self.bgr[f], self.ccam, self.dcam)
        return self.inten[f]

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
                frame = RefFrame(self.depth[fid], self.intensity(fid), np.array(W), self.dcam, self.p, self.c, self.depth[rid], self.intensity(rid),
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
    odo = RefOdometry(s, color=color, **track)
    for k, f in enumerate(ids):
        odo.step(f, pose_first=pose_first if k == 0 else None)
    return odo
