"""CPU tests of the photometric term of tracking through its restatement tests/track_color_ref.py (DESIGN.md §6p): the photometric row
against central differences, the frame intensity in the depth camera, a single textured plane (which depth alone cannot track), the
identity with the depth-only restatement at weight 0, the tiny scene's accuracy, and the golden fixture tests/golden/tiny_track_color.npz."""
import functools
import math
import os

import numpy as np
import pytest

import frames_ref
import track_color_ref as tc
import track_ref as tr
from test_odometry import live_grid
from test_track import _planes_view

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32


# ---- 1. the photometric row against central differences ----------------------------------------------------------------------------
def _affine_image(W, H, a, b, c):
    """I(x, y) = a + b x + c y: central differences are its gradient and bilinear sampling is exact, so the restated residual is a smooth
    function of the pose whose derivative the row must give"""
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return (a + b * xx + c * yy).astype(f32)


def _residual(xi, T, q, Im, cam, I):
    """I(pi(R'^T (q - t'))) - I_m in double for T' = [Rodrigues(w) | v] . T, I evaluated as the affine plane it samples"""
    Tn = np.array(tr.update(list(T), list(xi)))
    R, t = Tn[:9].reshape(3, 3), Tn[9:]
    xc = R.T @ (q - t)
    x = float(cam["fx"]) * xc[0] / xc[2] + float(cam["cx"])
    y = float(cam["fy"]) * xc[1] / xc[2] + float(cam["cy"])
    a, b, c = float(I[0, 0]), float(I[0, 1] - I[0, 0]), float(I[1, 0] - I[0, 0])
    return a + b * x + c * y - Im


def test_photometric_row_matches_central_differences():
    rng = np.random.default_rng(4)
    dcam = (64, 48, 50.0, 50.0, 31.5, 23.5)
    cam = tr.level_cams(dcam, 1)[0]
    c = tc.color_params(max_color_diff=10.0, min_color_gradient=0.0)
    for _ in range(20):
        I = _affine_image(64, 48, 0.3, rng.uniform(-0.01, 0.01), rng.uniform(-0.01, 0.01))
        gx, gy = tc.gradients(I)
        # a camera -> world pose and one model point in front of it
        w = rng.normal(size=3) * 0.3
        T = np.array(tr.update([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], list(w) + list(rng.normal(size=3) * 0.1)))
        xc = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.08, 0.08), rng.uniform(0.4, 0.8)])
        q = (T[:9].reshape(3, 3) @ xc + T[9:]).astype(f32)
        Im = f32(0.25)
        # a one-pixel prediction whose ray reproduces q: place q as the prediction's point via the float input pose = T itself
        rt_in = np.array(tr.inverse(list(T)), np.float64).astype(f32)
        xc32 = tr.xform(rt_in, rt_in[9:], [np.full((1, 1), q[k]) for k in range(3)])
        u = float(cam["fx"]) * float(xc32[0][0, 0]) / float(xc32[2][0, 0]) + float(cam["cx"])
        v = float(cam["fy"]) * float(xc32[1][0, 0]) / float(xc32[2][0, 0]) + float(cam["cy"])
        iu, iv = int(round(u)), int(round(v))
        # the model point the row uses is the prediction pixel's point: read it back from the restatement's own q
        pdepth = np.zeros((48, 64), f32)
        pdepth[iv, iu] = f32(xc32[2][0, 0])
        pint = np.full((48, 64), Im, f32)
        depth = np.full((48, 64), f32(xc32[2][0, 0]), f32)
        ok, J, r = tc.photo_rows(np.asarray(T).astype(f32), rt_in, cam, cam, 0, pdepth, pint, I, gx, gy, depth, f32(1.0), c)
        assert ok.sum() == 1
        k = np.argwhere(ok)[0]
        # the row's q, recomputed as the kernel forms it
        xn = (f32(iu) - cam["cx"]) / cam["fx"]
        yn = (f32(iv) - cam["cy"]) / cam["fy"]
        qk = np.array([(-((rt_in[j] * rt_in[9] + rt_in[3 + j] * rt_in[10]) + rt_in[6 + j] * rt_in[11])) +
                       pdepth[iv, iu] * ((rt_in[j] * xn + rt_in[3 + j] * yn) + rt_in[6 + j]) for j in range(3)], np.float64)
        T32 = np.asarray(T).astype(f32).astype(np.float64)
        assert r[k[0], k[1]] == pytest.approx(_residual(np.zeros(6), T32, qk, float(Im), cam, I), abs=1e-5)
        h = 1e-6
        num = np.array([(_residual(h * e, T32, qk, float(Im), cam, I) - _residual(-h * e, T32, qk, float(Im), cam, I)) / (2 * h)
                        for e in np.eye(6)])
        # float gradients of a plane with slope ~0.01 per pixel: agreement to ~1e-5 of the largest entry, every sign pinned
        assert np.allclose(J[k[0], k[1]], num, rtol=1e-3, atol=1e-4 * np.abs(num).max()), (J[k[0], k[1]], num)


# ---- 2. the frame intensity in the depth camera --------------------------------------------------------------------------------------
def test_frame_intensity_is_a_copy_for_equal_sizes_and_exact_for_a_2x_colour_camera():
    rng = np.random.default_rng(9)
    bgr = rng.integers(0, 256, size=(24, 32, 3), dtype=np.uint8)
    dcam = (32, 24, 32.0, 32.0, 15.5, 11.5)
    lum = frames_ref.intensity0(bgr)
    other = (32, 24, 40.0, 30.0, 16.0, 12.0)                      # equal size, other intrinsics: resizeDepth copies (Q51)
    assert tc.frame_intensity(bgr, other, dcam).tobytes() == lum.tobytes()
    up = np.repeat(np.repeat(bgr, 2, 0), 2, 1)                      # 2x nearest-upsampled colour, cx_c = 2 cx + 0.5
    ccam = (64, 48, 64.0, 64.0, 2 * 15.5 + 0.5, 2 * 11.5 + 0.5)
    assert tc.frame_intensity(up, ccam, dcam).tobytes() == lum.tobytes()


# ---- 3. a single textured plane ------------------------------------------------------------------------------------------------------
PLANE_DCAM = (64, 48, 50.0, 50.0, 31.5, 23.5)
# measured with the restatement: 2 mm in-plane and 0.5 deg about the normal are recovered to 0.001 deg and 0.01 mm
PLANE_TRANS_M = 5e-5
PLANE_ROT_DEG = 3e-3


def _texture(X, Y):
    """smooth at the pixel scale (periods of 20-25 px at 1 cm per pixel), so that bilinear sampling barely biases the residual"""
    return 0.5 + 0.3 * np.sin(2 * np.pi * X / 0.25) * np.cos(2 * np.pi * Y / 0.2)


def _down_pose(c, yaw_deg=0.0):
    """world -> camera of a camera at c looking straight down at the plane z = 0, rotated by yaw about the vertical"""
    a = math.radians(yaw_deg)
    Rz = np.array([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]])
    R = np.array([[1.0, 0, 0], [0, -1.0, 0], [0, 0, -1.0]]) @ Rz.T
    return np.concatenate([R.reshape(-1), -R @ np.asarray(c, np.float64)])


def _plane_intensity(rt, dcam):
    """the texture seen from rt (world -> camera) at every pixel, with its depth"""
    W, H, fx, fy, cx, cy = dcam
    depth, _ = _planes_view(rt, dcam, (2,))
    R, t = np.asarray(rt[:9], np.float64).reshape(3, 3), np.asarray(rt[9:], np.float64)
    o = -R.T @ t
    vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    d = np.stack([(uu - cx) / fx, (vv - cy) / fy, np.ones_like(uu, dtype=np.float64)], -1) @ R
    s = -o[2] / d[..., 2]
    P = o + s[..., None] * d
    return np.where(depth > 0, _texture(P[..., 0], P[..., 1]), 0).astype(f32), depth


def _plane_frames(**color):
    c_true = np.array([0.1, 0.05, 0.5])
    true = _down_pose(c_true)
    pose_in = _down_pose(c_true + np.array([0.0014, -0.0014, 0.0]), yaw_deg=0.5)
    inten, depth = _plane_intensity(true, PLANE_DCAM)
    pin = pose_in.astype(f32).astype(np.float64)
    pint, pdepth = _plane_intensity(pin, PLANE_DCAM)
    _, pnrm = _planes_view(pin, PLANE_DCAM, (2,))
    p = tr.params(num_levels=2, iterations=(10, 5))
    geo = tr.Frame(depth, pose_in, PLANE_DCAM, p, prediction=(pdepth, pnrm)).run()
    col = tc.ColorFrame(depth, inten, pose_in, PLANE_DCAM, p, tc.color_params(**color), prediction=(pdepth, pnrm, pint)).run()
    return geo, col, true


def test_single_textured_plane_tracks_with_colour_only():
    geo, col, true = _plane_frames()
    assert geo.status == 2                                          # §6n KT2: depth alone leaves three directions free
    assert col.status == 0 and col.iterations == 15, (col.status, col.iterations)
    r, t = tr.pose_errors([col.w2c], [true])
    print("textured plane: rot deg %.2e, centre m %.2e, photometric rows %d" % (r[0], t[0], col.last[0]))
    assert r[0] < PLANE_ROT_DEG and t[0] < PLANE_TRANS_M, (r, t)


# ---- 4. weight 0 is the depth-only restatement -----------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def tiny_fused():
    """the tiny scene fused from its colour frames at the true poses (the fusion oracle), as the march reads it, with its voxel colours,
    and the frames' intensity in the depth camera"""
    from intrinsic3d_b200.scene import config_scene
    from fusion_ref import FusionOracle, depth_range, scene_inputs
    s = config_scene("tiny")
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    lo, hi = depth_range(s)
    fo = FusionOracle(voxel_size=float(s["voxel_size"]), depth_min=lo, depth_max=hi)
    fo.integrate(dcam, depth, ccam, bgr, c2w, w2c)
    v = fo.volume()
    keep = v["weight"] > 0
    grid = live_grid(v, np.float32(s["voxel_size"]))
    inten = np.stack([tc.frame_intensity(b, ccam, dcam) for b in bgr])
    return s, dcam, depth, grid, v["rgb"][keep], inten, bgr


def test_weight_zero_equals_the_depth_only_restatement():
    s, dcam, depth, grid, rgb, inten, _ = tiny_fused()
    ids = [1, 4]
    start = tr.perturb(tr.aa_to_rt(s["poses_true"]), 1.0, 0.01, seed=5)[ids]
    it = dict(num_levels=2, iterations=(3, 2))
    geo = tr.track(grid, depth, ids, start, dcam, **it)
    col = tc.track(grid, rgb, depth, inten, ids, start, dcam, color=dict(weight=0.0), **it)
    for g, c in zip(geo, col):
        assert [g.status, g.iterations, g.correspondences] == [c.status, c.iterations, c.correspondences]
        assert g.sys.tobytes() == c.sys.tobytes() and np.array(g.w2c).tobytes() == np.array(c.w2c).tobytes()
        assert c.last[0] > 100                                        # the photometric rows are still formed and counted


# ---- 5. the golden fixture -------------------------------------------------------------------------------------------------------
def test_golden_fixture_matches_restatement():
    g = np.load(os.path.join(HERE, "golden", "tiny_track_color.npz"))
    grid = tr.rr.Grid(g["xyz"], g["sdf"], np.zeros(len(g["sdf"])), g["weight"], g["voxel_size"])
    ids = g["ids"].tolist()
    fr = tc.track(grid, g["rgb"], g["depth"], g["intensity"], ids, g["pose_in"], tuple(g["dcam"]), num_levels=int(g["num_levels"]),
                  iterations=g["iterations"].tolist())
    for k, f in enumerate(fr):
        assert f.pint.tobytes() == g["model_intensity"][k].tobytes()
        for l in range(int(g["num_levels"])):
            assert f.inten[l].tobytes() == g[f"intensity_{l}"][k].tobytes()
            assert f.grads[l][0].tobytes() == g[f"grad_x_{l}"][k].tobytes() and f.grads[l][1].tobytes() == g[f"grad_y_{l}"][k].tobytes()
        assert f.sys.tobytes() == g["sums"][k].tobytes() and f.sys_c.tobytes() == g["color_sums"][k].tobytes()
        assert [f.status, f.iterations, f.correspondences] == g["outcome"][k].tolist()
        assert [f.first[0], f.last[0]] == g["color_rows"][k].tolist()
        assert np.abs(np.array(f.w2c) - g["pose_out"][k]).max() < 1e-12
