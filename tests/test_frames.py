"""CPU checks of the keyframe blur score and image pyramid restatement (tests/frames_ref.py) and of the host-side keyframe selection and
keyframes file (intrinsic3d_b200/keyframes.py) against known answers."""
import math
import os

import numpy as np
import pytest

import frames_ref as R
from intrinsic3d_b200.keyframes import load_keyframes, save_keyframes, select_keyframes

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_frames.npz")


def _pattern(H=48, W=64, seed=0):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)


def test_grey_is_opencv_fixed_point():
    bgr = np.array([[[255, 255, 255], [0, 0, 0], [255, 0, 0], [0, 255, 0], [0, 0, 255], [10, 200, 30]]], np.uint8)
    assert R.grey_u8(bgr).tolist() == [[255, 0, 29, 150, 76, (1868 * 10 + 9617 * 200 + 4899 * 30 + 8192) >> 14]]


def test_constant_frame_scores_nan():
    bgr = np.full((20, 30, 3), 77, np.uint8)
    assert math.isnan(R.blur_score(bgr))


def test_stripes_along_x_score_one_minus_b_ver():
    """Stripes that run along x (constant along each row, changing from row to row): s_f_hor = 0, so b_hor is NaN and the score is
    1 - b_ver, because std::max(b_ver, NaN) = b_ver.  The transposed stripes have no vertical variation: b_ver is NaN and
    std::max(NaN, b_hor) = NaN, so the score is NaN.  The asymmetry is the reference's."""
    H, W = 24, 40
    rows = np.repeat((np.arange(H) % 5 * 50).astype(np.uint8)[:, None], W, axis=1)      # varies along y only
    bgr = np.repeat(rows[:, :, None], 3, axis=2)
    sfv, svv, sfh, svh = R.blur_sums(bgr)
    assert sfh == 0.0 and svh == 0.0 and sfv > 0.0
    b_ver = (sfv - svv) / sfv
    assert R.blur_score(bgr) == 1.0 - b_ver
    # the transpose varies along x only: b_ver is NaN and std::max(NaN, b_hor) is NaN
    assert math.isnan(R.blur_score(np.ascontiguousarray(bgr.transpose(1, 0, 2))))


def test_box_blurred_copy_scores_lower():
    bgr = _pattern()
    k = np.ones(5) / 5
    b = bgr.astype(np.float64)
    b = np.apply_along_axis(lambda r: np.convolve(r, k, "same"), 0, np.apply_along_axis(lambda r: np.convolve(r, k, "same"), 1, b))
    blurred = np.clip(np.rint(b), 0, 255).astype(np.uint8)
    assert R.blur_score(blurred) < R.blur_score(bgr)


def test_small_frames_refused():
    with pytest.raises(ValueError):
        R.blur_score(np.zeros((4, 10, 3), np.uint8))
    with pytest.raises(ValueError):
        R.pyr_down(np.zeros((2, 10), np.float32))
    with pytest.raises(ValueError):
        R.depth_down(np.zeros((10, 2), np.float32))
    assert R.pyr_down(np.ones((3, 3), np.float32)).shape == (1, 1)


def test_intensity0_formula():
    bgr = np.array([[[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 255]]], np.uint8)
    c = np.float32(1.0 / 255.0)
    one = np.float32(255) * c
    got = R.intensity0(bgr)[0]
    assert got[0] == one * np.float32(0.114) and got[1] == one * np.float32(0.587) and got[2] == one * np.float32(0.299)
    assert got[3] == (one * np.float32(0.114) + one * np.float32(0.587)) + one * np.float32(0.299)


@pytest.mark.parametrize("shape", [(8, 8), (121, 161), (5, 7), (3, 3)])
def test_pyrdown_constant_is_exact(shape):
    for v in (0.0, 0.25, 0.7071, 1.0):
        out = R.pyr_down(np.full(shape, v, np.float32))
        assert out.shape == (shape[0] // 2, shape[1] // 2)
        assert (out == np.float32(v)).all(), v


def test_pyrdown_matches_separable_5_tap_kernel():
    img = np.random.default_rng(1).random((11, 13)).astype(np.float32)
    k = np.array([1, 4, 6, 4, 1], np.float64) / 16
    pad = np.pad(img.astype(np.float64), 2, mode="reflect")             # numpy "reflect" = REFLECT_101
    full = np.array([[(k[:, None] * k[None, :] * pad[y:y + 5, x:x + 5]).sum() for x in range(13)] for y in range(11)])
    assert np.abs(R.pyr_down(img) - full[::2, ::2][:5, :6]).max() < 1e-6


def test_depth_holes():
    d = np.zeros((4, 6), np.float32)
    d[0, 0] = 1.2345678                                                 # block (0,0): one valid tap, kept exactly
    d[0:2, 2:4] = [[1.0, 2.0], [0.0, -1.0]]                             # block (0,1): taps 1, 2 valid; negative dropped
    d[2:4, 4:6] = [[0.1, 0.2], [0.3, 0.4]]                              # block (1,2): all four, in order
    out = R.depth_down(d)
    assert out.shape == (2, 3)
    assert out[0, 0] == np.float32(1.2345678)
    assert out[0, 1] == np.float32(1.5)
    s = ((np.float32(0.1) + np.float32(0.2)) + np.float32(0.3)) + np.float32(0.4)
    assert out[1, 2] == s / np.float32(4)
    assert out[0, 2] == 0.0 and out[1, 0] == 0.0 and out[1, 1] == 0.0   # all four taps invalid


def test_depth_odd_size():
    d = np.arange(1, 36, dtype=np.float32).reshape(5, 7)
    out = R.depth_down(d)
    assert out.shape == (2, 3)
    assert out[1, 2] == (((d[2, 4] + d[2, 5]) + d[3, 4]) + d[3, 5]) / np.float32(4)


def test_pyramid_chain_and_lum_given():
    bgr = np.stack([_pattern(21, 33, s) for s in range(2)])
    depth = np.random.default_rng(3).random((2, 21, 33)).astype(np.float32)
    L, D = R.pyramid(bgr, depth, 3)
    assert [x.shape for x in L] == [(2, 21, 33), (2, 10, 16), (2, 5, 8)]
    assert (L[2][1] == R.pyr_down(R.pyr_down(R.intensity0(bgr[1])))).all()
    assert (D[2][0] == R.depth_down(R.depth_down(depth[0]))).all()
    lum = np.full((2, 21, 33), 0.5, np.float32)
    L2, _ = R.pyramid(bgr, depth, 2, lum=lum)
    assert (L2[1] == np.float32(0.5)).all()


# ---- selectKeyframes -------------------------------------------------------------------------------------------------------------
def test_select_ties_go_to_the_earlier_frame():
    assert select_keyframes([0.3, 0.5, 0.5, 0.1], 4).tolist() == [False, True, False, False]


def test_select_nan_never_wins():
    assert select_keyframes([0.2, float("nan"), 0.3], 3).tolist() == [False, False, True]
    assert select_keyframes([float("nan"), 0.1], 2).tolist() == [False, True]


def test_select_all_non_positive_window_keeps_first():
    assert select_keyframes([-0.5, 0.0, float("nan"), 0.9, 0.8], 3).tolist() == [True, False, False, True, False]


def test_select_short_last_window():
    got = select_keyframes([0.1, 0.9, 0.2, 0.3, 0.7], 2)
    assert got.tolist() == [False, True, False, True, True]
    assert select_keyframes([0.4] * 41, 20).sum() == 3


def test_select_window_zero_refused():
    with pytest.raises(ValueError):
        select_keyframes([0.1, 0.2], 0)
    with pytest.raises(ValueError):
        select_keyframes([0.1, 0.2], -3)


# ---- keyframes file --------------------------------------------------------------------------------------------------------------
def test_reference_file_with_nan_loads_as_the_reference_would(tmp_path):
    p = tmp_path / "keyframes.txt"
    p.write_text("20\n0.812345 1\n\n0.500000 0\nnan 0\n0.900000 1\n")
    window, scores, flags = load_keyframes(str(p))
    assert window == 20
    assert scores.tolist() == [0.812345, 0.5]
    assert flags.tolist() == [True, False]


def test_bad_flag_stops_the_load(tmp_path):
    p = tmp_path / "k.txt"
    p.write_text("5\n0.1 1\n0.2 2\n0.3 1\n")
    assert load_keyframes(str(p))[1].tolist() == [0.1]
    p.write_text("\n0.1 1\n")
    with pytest.raises(ValueError):
        load_keyframes(str(p))


def test_save_load_round_trip(tmp_path):
    scores = np.array([0.1234564, 0.75, 1.0, 0.0, -0.25])
    sel = select_keyframes(scores, 2)
    p = tmp_path / "k.txt"
    save_keyframes(str(p), scores, sel, 2)
    text = p.read_text().splitlines()
    assert text[0] == "2" and text[1] == "0.123456 0" and text[2] == "0.750000 1"
    window, s2, f2 = load_keyframes(str(p))
    assert window == 2 and f2.tolist() == sel.tolist()
    assert np.abs(s2 - scores).max() <= 5e-7
    # a NaN score truncates the reload there, as in the reference
    save_keyframes(str(p), [0.5, float("nan"), 0.7], [True, False, True], 20)
    assert "nan 0" in p.read_text()
    assert load_keyframes(str(p))[1].tolist() == [0.5]


def test_golden_fixture():
    g = np.load(GOLDEN)
    bgr, depth = g["bgr"], g["depth"]
    scores = R.blur_scores(bgr)
    assert np.abs(scores - g["scores"]).max() <= 1e-13
    assert g["scores"][1] < g["scores"][0] and g["scores"][1] < g["scores"][2]         # the box-blurred frame is the least sharp
    assert (select_keyframes(scores, int(g["window"])) == g["selection"]).all()
    L, D = R.pyramid(bgr, depth, 3)
    for k, a in (("lum0", L[0]), ("lum1", L[1]), ("lum2", L[2]), ("depth1", D[1]), ("depth2", D[2])):
        assert a.tobytes() == g[k].tobytes(), k
