"""numpy restatement of the photometric term of tracking (intrinsic3d_b200/csrc/i3d_track.cuh, DESIGN.md §6p).

Built on tests/track_ref.py (the geometric rows, sums and solve), tests/render_ref.py (the march) and tests/frames_ref.py /
tests/sensor_ref.py (the intensity rule, pyrDown and resizeDepth), which it leaves as they are.  Every float operation is one numpy float32
operation and every double operation one float64 operation, in the device's order, so the model intensity, frame intensity and gradient
planes are byte-equal and the photometric sums are the device's bit for bit.
"""
from __future__ import annotations

import numpy as np

import frames_ref
import render_ref as rr
import sensor_ref
import track_ref as tr

f32 = np.float32
INV255 = f32(1.0 / 255.0)
DEFAULTS = dict(weight=(0.05, 0.05, 0.05, 0.05), max_color_diff=0.1, min_color_gradient=0.01)


def color_params(**over):
    c = dict(DEFAULTS)
    c.update(over)
    w = c["weight"]
    w = [float(w)] * 4 if np.ndim(w) == 0 else list(w) + [0.0] * (4 - len(w))
    c["weight"] = tuple(f32(x) for x in w)
    c["max_color_diff"] = f32(c["max_color_diff"])
    c["min_color_gradient"] = f32(c["min_color_gradient"])
    return c


def voxel_intensity(rgb):
    """rd_float(uchar4): the frame store's level-0 rule on voxel colours R, G, B [n, 3] -> float32 [n]"""
    c = np.asarray(rgb, np.uint8).astype(f32) * INV255
    return (c[:, 2] * f32(0.114) + c[:, 1] * f32(0.587)) + c[:, 0] * f32(0.299)


def model_intensity(grid, rgb, view):
    """The model intensity plane [H, W] of a march view (render_ref.render_view): at a hit the trilinear blend of the corners'
    intensities in the cube of the hit point o + s_hit dn (rd_point), 0 elsewhere"""
    H, W = view["depth"].shape
    out = np.zeros(H * W, f32)
    hit = view["hit"].ravel()
    if hit.any():
        o, dn = view["ray"]
        dn = dn.reshape(-1, 3)[hit]
        s = view["s_hit"].ravel()[hit]
        p = o[None, :] + s[:, None] * dn
        c, f, ok = grid.cube(p)
        assert ok.all()
        out[hit] = rr.Grid.trilinear(voxel_intensity(rgb), c, f)
    return out.reshape(H, W)


def frame_intensity(bgr, ccam, dcam):
    """The stored colour frame's level-0 intensity in the depth camera: k_frames_lum0, then resizeDepth from the colour camera (a copy when
    the sizes agree, Q51)"""
    return sensor_ref.resize_depth(frames_ref.intensity0(np.asarray(bgr, np.uint8)), ccam, dcam)


def intensity_pyramid(inten0, levels):
    out = [np.asarray(inten0, f32)]
    for _ in range(1, levels):
        out.append(frames_ref.pyr_down(out[-1]))
    return out


def gradients(I):
    """k_track_grad: FM(0.5, I[+1] - I[-1]) on 1..W-2 x 1..H-2, 0 on the border"""
    I = np.asarray(I, f32)
    gx, gy = np.zeros_like(I), np.zeros_like(I)
    gx[1:-1, 1:-1] = f32(0.5) * (I[1:-1, 2:] - I[1:-1, :-2])
    gy[1:-1, 1:-1] = f32(0.5) * (I[2:, 1:-1] - I[:-2, 1:-1])
    return gx, gy


def _bilinear(P, x0, y0, fx, fy):
    r0 = P[y0, x0] + fx * (P[y0, x0 + 1] - P[y0, x0])
    r1 = P[y0 + 1, x0] + fx * (P[y0 + 1, x0 + 1] - P[y0 + 1, x0])
    return r0 + fy * (r1 - r0)


def photo_rows(Tf, rt_in, cam0, cam, l, pdepth, pint, I, gx, gy, depth_l, max_distance, c):
    """k_track_photo_rows of one frame at level l: (ok [H_l, W_l], J [H_l, W_l, 6], r [H_l, W_l]) in double"""
    H, W = I.shape
    step = 1 << l
    vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    iu, iv = uu * step, vv * step
    zm = pdepth[iv, iu]
    Im = pint[iv, iu]
    ok = zm > 0
    R0 = np.asarray(rt_in, f32)
    Tf = np.asarray(Tf, f32)
    with np.errstate(all="ignore"):
        xn = (iu.astype(f32) - cam0["cx"]) / cam0["fx"]
        yn = (iv.astype(f32) - cam0["cy"]) / cam0["fy"]
        q = []
        for k in range(3):
            o = -((R0[k] * R0[9] + R0[3 + k] * R0[10]) + R0[6 + k] * R0[11])
            dr = (R0[k] * xn + R0[3 + k] * yn) + R0[6 + k]
            q.append(o + zm * dr)
        e = [q[k] - Tf[9 + k] for k in range(3)]
        xc = [(Tf[d] * e[0] + Tf[3 + d] * e[1]) + Tf[6 + d] * e[2] for d in range(3)]
        ok &= xc[2] > 0
        x = cam["fx"] * (xc[0] / xc[2]) + cam["cx"]
        y = cam["fy"] * (xc[1] / xc[2]) + cam["cy"]
        ok &= (x >= f32(1.0)) & (x < f32(W - 2)) & (y >= f32(1.0)) & (y < f32(H - 2))
        xs, ys = np.where(ok, x, f32(1.0)), np.where(ok, y, f32(1.0))
        ou = np.trunc(xs + f32(0.5)).astype(np.int64)
        ov = np.trunc(ys + f32(0.5)).astype(np.int64)
        d = depth_l[ov, ou]
        ok &= (d > 0) & (np.abs(d - xc[2]) <= max_distance)
        xf, yf = np.floor(xs), np.floor(ys)
        x0, y0 = xf.astype(np.int64), yf.astype(np.int64)
        fx, fy = xs - xf, ys - yf
        If = _bilinear(I, x0, y0, fx, fy)
        gxv = _bilinear(gx, x0, y0, fx, fy)
        gyv = _bilinear(gy, x0, y0, fx, fy)
        rc = If - Im
        ok &= (np.abs(rc) <= c["max_color_diff"]) & ((gxv * gxv + gyv * gyv) >= c["min_color_gradient"] * c["min_color_gradient"])
        gfx, gfy = gxv * cam["fx"], gyv * cam["fy"]
        gc = [gfx / xc[2], gfy / xc[2], -((gfx * xc[0] + gfy * xc[1]) / (xc[2] * xc[2]))]
        gw = tr.xform(Tf, None, gc)
    g = [np.where(ok, gw[k], 0).astype(np.float64) for k in range(3)]
    qd = [np.where(ok, q[k], 0).astype(np.float64) for k in range(3)]
    J = np.stack([g[1] * qd[2] - g[2] * qd[1], g[2] * qd[0] - g[0] * qd[2], g[0] * qd[1] - g[1] * qd[0],
                  np.where(ok, -g[0], 0.0), np.where(ok, -g[1], 0.0), np.where(ok, -g[2], 0.0)], -1)
    r = np.where(ok, rc, 0).astype(np.float64)
    return ok, J, r


def combine(Sg, Sc, weight):
    """k_track_combine: A = A_g + lam^2 A_c, b likewise (entries 0..26; the geometric ones for lam = 0), geometric r^2 and rows"""
    lam2 = float(weight) * float(weight)
    S = np.array(Sg, np.float64)
    if lam2 != 0.0:
        S[:27] = Sg[:27] + lam2 * Sc[:27]
    return S


class ColorFrame(tr.Frame):
    """One frame's joint depth and colour problem: track_ref.Frame plus the model intensity at the input pose, the frame intensity
    pyramid and its gradients; every system is combine(geometric, photometric)."""

    def __init__(self, depth0, inten0, pose_in, dcam, p, c, grid=None, rgb=None, prediction=None):
        initial = None
        if prediction is None:
            # the march at the input pose once: depth, normal and the model intensity (track_ref.predict's view)
            cam0 = tr.level_cams(dcam, 1)[0]
            cam = dict(fx=cam0["fx"], fy=cam0["fy"], cx=cam0["cx"], cy=cam0["cy"], d=np.zeros(5, f32))
            d0 = np.asarray(depth0, f32)
            view = rr.render_view(grid, np.asarray(pose_in, np.float64).astype(f32), cam, cam0["W"], cam0["H"], photometric=False)
            prediction = (view["depth"], view["normal"], model_intensity(grid, rgb, view))
            initial = rr.stats(view, d0, np.zeros_like(d0))
        super().__init__(depth0, pose_in, dcam, p, prediction=prediction[:2])
        self.initial = initial
        self.c = c
        self.pint = np.asarray(prediction[2], f32)
        self.inten = intensity_pyramid(inten0, p["num_levels"])
        self.grads = [gradients(I) for I in self.inten]
        self.sys_c = np.zeros(tr.VALS)
        self.first = None
        self.last = (0, 0.0)

    def photo_system(self, l):
        ok, J, r = photo_rows(self.Tf(), self.rt_in, self.cams[0], self.cams[l], l, self.pdepth, self.pint, self.inten[l], *self.grads[l],
                              self.depth[l], self.p["max_distance"], self.c)
        return tr.tile_sums(tr.values(J, r, ok))

    def system(self, l):
        Sg = super().system(l)
        Sc = self.photo_system(l)
        self.sys_c = Sc
        rec = (int(Sc[28]), float(Sc[27]))
        if self.first is None:
            self.first = rec
        self.last = rec
        return combine(Sg, Sc, self.c["weight"][l])


def track(grid, rgb, depth_frames, inten_frames, ids, pose_in, dcam, color=None, **over):
    """i3d_track_sensor_frames_rgbd restated: one ColorFrame per id (run), in call order.  inten_frames: the frames' intensity in the depth
    camera (frame_intensity)."""
    p = tr.params(**over)
    c = color_params(**(color or {}))
    return [ColorFrame(depth_frames[f], inten_frames[f], pose_in[k], dcam, p, c, grid=grid, rgb=rgb).run() for k, f in enumerate(ids)]
