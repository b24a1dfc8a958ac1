"""Known answers of tests/sensor_ref.py, the numpy restatement of resizeDepth + interpolate<float> that checks k_resize_depth, and the
golden fixture tests/golden/tiny_sensor.npz."""
import os

import numpy as np

import sensor_ref as S

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _depth(W, H, seed=0, holes=0.2):
    rng = np.random.default_rng(seed)
    d = (0.5 + rng.random((H, W))).astype(F32)
    d[rng.random((H, W)) < holes] = 0.0
    return d


def test_equal_sizes_copy_whatever_the_intrinsics():
    d = _depth(40, 30)
    cam = (40, 30, 50.0, 52.0, 19.5, 14.5)
    for other in ((40, 30, 80.0, 30.0, 3.0, 27.0), S.color_cameras(cam)["same_size"]):
        out = S.resize_depth(d, cam, other)
        assert out.dtype == F32 and out.tobytes() == d.tobytes()


# u = 0.625 x - 3.9375, v = 0.625 y - 1.9375: columns 5..69 and rows 2..50 have a tap in range with a positive weight; column 4
# (u = -1.4375) has a tap in range but no weight inside the plane
IN_CAM = (40, 30, 50.0, 50.0, 20.0, 15.0)
OUT_CAM = (80, 60, 80.0, 80.0, 38.3, 27.1)


def test_constant_plane_stays_constant_where_the_tap_is_in_range():
    c = F32(1.7)
    out = S.resize_depth(np.full((30, 40), c, F32), IN_CAM, OUT_CAM)
    inside = np.zeros((60, 80), bool)
    inside[2:51, 5:70] = True
    assert (out[~inside] == 0).all()
    assert np.abs(out[inside] - c).max() <= 2 * np.spacing(c)
    # a power of two makes every product and sum exact up to the reordering of the weight sum: within one ulp
    out2 = S.resize_depth(np.full((30, 40), F32(2.0), F32), IN_CAM, OUT_CAM)
    assert np.abs(out2[inside] - F32(2.0)).max() <= np.spacing(F32(2.0))


def test_zero_pixel_lowers_its_resized_neighbours():
    d = np.full((30, 40), F32(2.0), F32)
    d[14, 20] = 0.0
    out = S.resize_depth(d, IN_CAM, OUT_CAM)
    ref = S.resize_depth(np.full((30, 40), F32(2.0), F32), IN_CAM, OUT_CAM)
    lowered = out < ref - F32(1e-3)
    ys, xs = np.nonzero(lowered)
    # every output pixel whose bilinear footprint [u0, u0 + 1] x [v0, v0 + 1] holds column 20 / row 14 (Q50), and no other one
    assert 0 < lowered.sum() <= 16
    u = 0.625 * xs - 3.9375
    v = 0.625 * ys - 1.9375
    assert (np.abs(u - 20) < 1).all() and (np.abs(v - 14) < 1).all()
    assert (out[~lowered] == ref[~lowered]).all()
    assert (out[lowered] > 0).any()                                  # pulled towards 0, not dropped


def test_band_left_of_column_zero_and_the_right_edge():
    d = np.tile(np.arange(1, 9, dtype=F32), (4, 1))                  # column j holds j + 1
    cam = (8, 4, 1.0, 1.0, 0.0, 0.0)
    # u = x - cx: cx 0.75 -> u(0) = -0.75, cx 0.5 -> u(0) = -0.5 (both in (-1, -0.5]: column 0); cx 1.25 -> u(0) = -1.25 (no weight: 0)
    for cx, first in ((0.75, 1.0), (0.5, 1.0), (1.25, 0.0)):
        out = S.resize_depth(d, cam, (12, 4, 1.0, 1.0, cx, 0.0))
        assert (out[:, 0] == F32(first)).all(), (cx, out[0])
        u = np.arange(12) - cx
        assert (out[:, u >= 7.5] == 0).all()                          # u >= Wd - 0.5: the tap is column Wd, outside
        assert (out[:, (u > -1) & (u < 7.5)] > 0).all()
    out = S.resize_depth(d, cam, (12, 4, 1.0, 1.0, 0.5, 0.0))
    assert out[0, 8] == 0 and out[0, 7] == F32(7.5)                   # u = 7.5 gives 0; u = 6.5 blends columns 6 and 7


def test_batches_and_shapes():
    d = np.stack([_depth(40, 30, seed=k) for k in range(3)])
    out = S.resize_depth(d, IN_CAM, OUT_CAM)
    assert out.shape == (3, 60, 80) and out.dtype == F32
    assert out[1].tobytes() == S.resize_depth(d[1], IN_CAM, OUT_CAM).tobytes()


def test_golden_fixture():
    g = np.load(os.path.join(ROOT, "tests", "golden", "tiny_sensor.npz"))
    dcam, ccam = tuple(g["depth_cam"]), tuple(g["color_cam"])
    dcam = (int(dcam[0]), int(dcam[1])) + dcam[2:]
    ccam = (int(ccam[0]), int(ccam[1])) + ccam[2:]
    assert ccam == S.color_cameras(dcam)["color_x2"]
    out = S.resize_depth(g["depth"], dcam, ccam)
    assert out.tobytes() == g["resized"].tobytes()
    assert (out > 0).sum() > 10000 and (out == 0).sum() > 10000
