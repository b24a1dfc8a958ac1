"""numpy float32 restatement of the keyframe blur score and the RGB-D image pyramid (intrinsic3d_b200/csrc/i3d_frames.cuh, DESIGN.md §6i).

Every float operation is a separate float32 numpy operation (no contraction), in the order the kernels fix, so the kernels' planes match it
bit for bit.  The four plane sums of the blur score are float64 numpy sums of the exactly converted floats; the kernels sum in another fixed
order, so scores agree to the last bits of a double sum, not bit for bit.

Reference steps: KeyframeSelection::estimateBlur / estimateBlurCrete (src/keyframe_selection.cpp:219-310) and Pyramid::create /
downsample / downsampleDepth (src/rgbd/pyramid.cpp:59-166)."""
import numpy as np

F32 = np.float32
INV255 = F32(1.0 / 255.0)
BOX_W = F32(1.0 / 9.0)


def reflect101(i, n):
    """BORDER_REFLECT_101 index map, one reflection (valid for -n < i < 2n - 1)."""
    i = np.asarray(i)
    return np.where(i < 0, -i, np.where(i >= n, 2 * n - 2 - i, i))


def grey_u8(bgr):
    """OpenCV's fixed-point 8-bit BGR2GRAY: (1868 B + 9617 G + 4899 R + 8192) >> 14.  bgr uint8 [..., 3]."""
    b = bgr[..., 0].astype(np.int32)
    g = bgr[..., 1].astype(np.int32)
    r = bgr[..., 2].astype(np.int32)
    return ((1868 * b + 9617 * g + 4899 * r + 8192) >> 14).astype(np.uint8)


def _box9(g, axis):
    """9-tap box filter along `axis`, taps added k = 0..8 as s = s + w * x[k] with the product rounded separately."""
    n = g.shape[axis]
    s = np.zeros_like(g)
    for k in range(9):
        idx = reflect101(np.arange(n) - 4 + k, n)
        s = s + BOX_W * np.take(g, idx, axis=axis)
    return s


def _absdiff(a, axis):
    d = np.zeros_like(a)
    if axis == 0:
        d[1:] = np.abs(a[1:] - a[:-1])
    else:
        d[:, 1:] = np.abs(a[:, 1:] - a[:, :-1])
    return d


def blur_sums(bgr):
    """(s_f_ver, s_v_ver, s_f_hor, s_v_hor) of one frame, bgr uint8 [H, W, 3]."""
    H, W = bgr.shape[:2]
    if H < 5 or W < 5:
        raise ValueError("blur score needs at least 5 px on each axis")
    g = grey_u8(bgr).astype(F32) * INV255
    out = []
    for axis in (0, 1):
        df = _absdiff(g, axis)
        db = _absdiff(_box9(g, axis), axis)
        v = np.maximum(F32(0.0), df - db)
        out += [float(df.astype(np.float64).sum()), float(v.astype(np.float64).sum())]
    return tuple(out)


def blur_score(bgr):
    """KeyframeSelection::estimateBlur of one BGR frame: 1 - std::max(b_ver, b_hor), b = (s_f - s_v) / s_f, NaN kept as the reference
    keeps it (std::max(a, NaN) is a, std::max(NaN, b) is NaN)."""
    s_f_ver, s_v_ver, s_f_hor, s_v_hor = blur_sums(bgr)
    with np.errstate(invalid="ignore", divide="ignore"):
        b_ver = (np.float64(s_f_ver) - s_v_ver) / np.float64(s_f_ver)
        b_hor = (np.float64(s_f_hor) - s_v_hor) / np.float64(s_f_hor)
    m = b_hor if b_ver < b_hor else b_ver
    return float(1.0 - m)


def blur_scores(bgr):
    """bgr uint8 [F, H, W, 3] -> float64 [F]."""
    return np.array([blur_score(f) for f in bgr], np.float64)


def intensity0(bgr):
    """Level-0 intensity from BGR: c = float(u8) * float(1/255) per channel, then (B 0.114 + G 0.587) + R 0.299.  [..., H, W, 3] -> float32."""
    c = bgr.astype(F32) * INV255
    return (c[..., 0] * F32(0.114) + c[..., 1] * F32(0.587)) + c[..., 2] * F32(0.299)


def _pyr5(a, b, c, d, e):
    """((6 c + 4 (b + d)) + a) + e."""
    return ((F32(6.0) * c + F32(4.0) * (b + d)) + a) + e


def pyr_down(img):
    """cv::pyrDown of one float plane [H, W] to (W // 2, H // 2), REFLECT_101: row pass stored as float, column pass, times 1/256."""
    H, W = img.shape
    if H < 3 or W < 3:
        raise ValueError("pyrDown needs a source of at least 3 px on each axis")
    Wd, Hd = W // 2, H // 2
    cx = [reflect101(2 * np.arange(Wd) + k, W) for k in range(-2, 3)]
    rows = _pyr5(*(img[:, c] for c in cx))                      # [H, Wd]
    cy = [reflect101(2 * np.arange(Hd) + k, H) for k in range(-2, 3)]
    return _pyr5(*(rows[c, :] for c in cy)) * F32(1.0 / 256.0)


def depth_down(depth):
    """Pyramid::downsampleDepth: taps (2y,2x), (2y,2x+1), (2y+1,2x), (2y+1,2x+1) in that order, only taps > 0, sum / float(cnt); 0 without
    a valid tap."""
    H, W = depth.shape
    if H < 3 or W < 3:
        raise ValueError("downsampleDepth needs a source of at least 3 px on each axis")
    Hd, Wd = H // 2, W // 2
    s = np.zeros((Hd, Wd), F32)
    cnt = np.zeros((Hd, Wd), np.int32)
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        d = depth[dy:2 * Hd:2, dx:2 * Wd:2]
        ok = d > F32(0.0)
        s = np.where(ok, s + d, s)
        cnt += ok
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(cnt > 0, s / cnt.astype(F32), F32(0.0)).astype(F32)


def pyramid(bgr, depth, levels, lum=None):
    """Levels 0..levels-1 of every frame, built as a chain: lists of float32 [F, H_l, W_l] intensity and depth planes."""
    lum0 = intensity0(bgr) if lum is None else np.asarray(lum, F32)
    L, D = [lum0.astype(F32)], [np.asarray(depth, F32)]
    for _ in range(1, levels):
        L.append(np.stack([pyr_down(x) for x in L[-1]]))
        D.append(np.stack([depth_down(x) for x in D[-1]]))
    return L, D
