"""numpy float32 restatement of resizeDepth + interpolate<float> (src/rgbd/processing.cpp:129-183, 236-291), the checker of k_resize_depth
(intrinsic3d_b200/csrc/i3d_frames.cuh, DESIGN.md §6l).  It shares no code with the kernel.

Every float operation is a separate float32 numpy operation (no contraction), in the order the contract fixes, so the kernel's planes
match it bit for bit.  Two quirks of the reference are kept: a zero-depth tap counts with its weight (Q50), and planes of equal size are
copied whatever the intrinsics (Q51)."""
import numpy as np

F32 = np.float32


def color_cameras(depth_cam):
    """The colour cameras the sensor tests pair with a depth camera (W, H, fx, fy, cx, cy): twice the size with its own intrinsics (the
    fusion tests' colour camera), the same size with other intrinsics (a copy, Q51), and 1.5x with a shifted principal point, so that
    the taps of the left columns and the bottom rows fall outside the depth plane."""
    W, H, fx, fy, cx, cy = depth_cam
    return {"color_x2": (2 * W, 2 * H, 2.1 * fx, 1.9 * fy, 2 * cx + 3.5, 2 * cy - 2.0),
            "same_size": (W, H, 1.1 * fx, 0.9 * fy, cx + 5.0, cy - 3.0),
            "x1.5_shifted": (3 * W // 2, 3 * H // 2, 1.5 * fx, 1.5 * fy, 1.5 * cx + 20.0, 1.5 * cy - 15.0)}


def _coords(n, out_c, out_f, in_f, in_c):
    """u (or v) of every output column (or row): ((float(x) - out_c) * FD(1, out_f)) * in_f + in_c."""
    inv = F32(1.0) / F32(out_f)
    return (F32(in_f) * ((np.arange(n).astype(F32) - F32(out_c)) * inv)) + F32(in_c)


def resize_depth(depth, in_cam, out_cam):
    """resizeDepth of one plane [Hd, Wd] or of frames [F, Hd, Wd] from in_cam to out_cam, each (W, H, fx, fy, cx, cy)."""
    depth = np.asarray(depth, F32)
    if depth.ndim == 3:
        return np.stack([resize_depth(d, in_cam, out_cam) for d in depth]) if len(depth) else np.zeros((0, out_cam[1], out_cam[0]), F32)
    Hi, Wi = depth.shape
    Wo, Ho = int(out_cam[0]), int(out_cam[1])
    assert (Wi, Hi) == (int(in_cam[0]), int(in_cam[1]))
    if (Wo, Ho) == (Wi, Hi):
        return depth.copy()
    u = np.broadcast_to(_coords(Wo, out_cam[4], out_cam[2], in_cam[2], in_cam[4])[None, :], (Ho, Wo))
    v = np.broadcast_to(_coords(Ho, out_cam[5], out_cam[3], in_cam[3], in_cam[5])[:, None], (Ho, Wo))
    tu, tv = u + F32(0.5), v + F32(0.5)
    # (int)(t) truncates toward zero, so it lies in [0, n) exactly when -1 < t < n
    tap = (tu > F32(-1.0)) & (tu < F32(Wi)) & (tv > F32(-1.0)) & (tv < F32(Hi))
    with np.errstate(invalid="ignore"):
        x0 = np.where(tap, np.floor(u), 0).astype(np.int64)
        y0 = np.where(tap, np.floor(v), 0).astype(np.int64)
    x1, y1 = x0 + 1, y0 + 1
    wx1 = u - x0.astype(F32)
    wy1 = v - y0.astype(F32)
    wx0, wy0 = F32(1.0) - wx1, F32(1.0) - wy1
    wx0 = np.where((x0 < 0) | (x0 >= Wi), F32(0.0), wx0)
    wx1 = np.where((x1 < 0) | (x1 >= Wi), F32(0.0), wx1)
    wy0 = np.where((y0 < 0) | (y0 >= Hi), F32(0.0), wy0)
    wy1 = np.where((y1 < 0) | (y1 >= Hi), F32(0.0), wy1)
    w00, w10, w01, w11 = wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1
    sw = ((w00 + w10) + w01) + w11
    s = np.zeros((Ho, Wo), F32)
    for w, yy, xx in ((w00, y0, x0), (w01, y1, x0), (w10, y0, x1), (w11, y1, x1)):
        ok = w > F32(0.0)
        d = depth[np.where(ok, yy, 0), np.where(ok, xx, 0)]
        s = np.where(ok, s + d * w, s)
    ok = tap & (sw > F32(0.0))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(ok, s / np.where(ok, sw, F32(1.0)), F32(0.0)).astype(F32)
    return np.where(r == F32(0.0), F32(0.0), r).astype(F32)     # the reference leaves +0 where the result is 0
