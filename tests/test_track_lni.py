"""CPU tests of the locally normalised intensity of the _ref calls through its restatement tests/track_lni_ref.py (DESIGN.md §6r): known
answers of the normalisation (a constant plane, clipped border windows), its invariance to a gain and an offset, the invariance to the
synthetic frames' per-frame colour modulation on the tiny scene, the restated LNI odometry on the dense tiny sequence, and the golden
fixture tests/golden/tiny_track_lni.npz."""
import os

import numpy as np
import pytest

import track_color_ref as tc
import track_lni_ref as tl
import track_ref as tr
import track_reference_ref as trr
from test_odometry import ANCHORED, dense_tiny

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32


def _window_stats(I, x, y, r):
    """float64 mean and variance of the (2r+1)^2 window of (x, y) clipped to the plane, and its pixel count"""
    H, W = I.shape
    w = I[max(y - r, 0):min(y + r, H - 1) + 1, max(x - r, 0):min(x + r, W - 1) + 1].astype(np.float64)
    return w.mean(), w.var(), w.size


# ---- 1. the normalisation ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value", [0.37, 0.5, 1.0 / 3.0, 0.0])
def test_a_constant_plane_gives_exactly_zero(value):
    for r in (1, 3, 8):
        out = tl.local_norm(np.full((13, 21), value, f32), r, 0.01)
        assert out.tobytes() == np.zeros((13, 21), f32).tobytes(), (value, r)


def test_a_constant_window_gives_zero_beside_texture():
    rng = np.random.default_rng(1)
    I = np.full((30, 40), f32(0.41), f32)
    I[:, 25:] = rng.uniform(0, 1, (30, 15)).astype(f32)
    out = tl.local_norm(I, 3, 0.01)
    assert (out[:, :22] == 0).all() and (out[:, 22:] != 0).all()


def test_clipped_border_windows_known_answer():
    rng = np.random.default_rng(2)
    I = rng.uniform(0, 1, (17, 23)).astype(f32)
    for r, eps in ((1, 0.01), (4, 0.01), (8, 0.2)):
        out = tl.local_norm(I, r, eps)
        for (x, y, n) in ((0, 0, (r + 1) ** 2), (22, 16, (r + 1) ** 2), (0, 8, (r + 1) * min(2 * r + 1, 17)), (11, 0, min(2 * r + 1, 23) * (r + 1))):
            mu, var, size = _window_stats(I, x, y, r)
            assert size == n, (r, x, y)
            want = (I[y, x] - mu) / np.sqrt(var + eps * eps)
            assert abs(out[y, x] - want) <= 1e-5 * max(1.0, abs(want)), (r, x, y, out[y, x], want)


def test_gain_and_offset_cancel():
    rng = np.random.default_rng(3)
    I = rng.uniform(0.1, 0.9, (40, 50)).astype(f32)
    base = tl.local_norm(I, 5, 1e-4).astype(np.float64)
    for a, b in ((1.7, 0.2), (0.6, -0.05), (1.05, 0.01)):
        out = tl.local_norm((f32(a) * I + f32(b)).astype(f32), 5, 1e-4)
        assert np.abs(out - base).max() <= 2e-4, (a, b, np.abs(out - base).max())


def test_pyramid_levels_come_from_the_raw_levels():
    rng = np.random.default_rng(4)
    I = rng.uniform(0, 1, (48, 64)).astype(f32)
    c = tl.color_params(norm_radius=2, norm_eps=0.01)
    raw = tc.intensity_pyramid(I, 3)
    got = tl.pyramid(I, 3, c)
    for l in range(3):
        assert got[l].tobytes() == tl.local_norm(raw[l], 2, 0.01).tobytes()
    assert [a.tobytes() for a in tl.pyramid(I, 3, tl.color_params(norm_radius=0))] == [a.tobytes() for a in raw]


# ---- 2. the invariance to the frames' colour modulation --------------------------------------------------------------------------
def _residual_ratio(bgr, s, r):
    """rms(I_f - model) / std(I_f) per level over frames 1..11 of the dense tiny sequence, each modelled from frame k - 1, both at their
    true poses, with the frame's own depth as the prediction"""
    from fusion_ref import scene_inputs
    dcam, depth, ccam, _, _, _ = scene_inputs(s)
    true = tr.aa_to_rt(s["poses_true"]).astype(f32)
    L = 3
    cams = tr.level_cams(dcam, L)
    c = tl.color_params(norm_radius=r, norm_eps=0.01)
    acc = np.zeros((L, 2))
    for k in range(1, 12):
        Pf = tl.pyramid(tc.frame_intensity(bgr[k], ccam, dcam), L, c)
        Pr = tl.pyramid(tc.frame_intensity(bgr[k - 1], ccam, dcam), L, c)
        Dr = tr.pyramid(depth[k - 1], L)
        for l in range(L):
            m = trr.ref_model(true[k], cams[0], cams[l], l, depth[k], true[k - 1], Pr[l], Dr[l], f32(0.05))
            ok = np.isfinite(m)
            acc[l] += [np.mean((Pf[l][ok] - m[ok]).astype(np.float64) ** 2), np.var(Pf[l].astype(np.float64))]
    return np.sqrt(acc[:, 0] / acc[:, 1])


def test_lni_removes_the_colour_modulation_on_the_tiny_scene():
    """raw intensity: the modulated frames' residual is 16-22 % above clean luminance's; LNI r = 5: within 1 % at every level"""
    from fusion_ref import scene_inputs
    s = dense_tiny(72)
    bgr = scene_inputs(s)[3]
    clean = np.repeat(np.clip(np.rint(np.asarray(s["lum"], f32) * f32(255.0)), 0, 255).astype(np.uint8)[..., None], 3, axis=-1)
    raw_mod, raw_clean = _residual_ratio(bgr, s, 0), _residual_ratio(clean, s, 0)
    lni_mod, lni_clean = _residual_ratio(bgr, s, 5), _residual_ratio(clean, s, 5)
    print("rms(r)/std(I) by level: raw %s vs clean %s; LNI %s vs clean %s" % (raw_mod.round(3), raw_clean.round(3), lni_mod.round(3),
                                                                           lni_clean.round(3)))
    assert (raw_mod > 1.1 * raw_clean).all()
    assert (np.abs(lni_mod / lni_clean - 1) < 0.01).all()


# ---- 3. the LNI odometry loop -------------------------------------------------------------------------------------------------------
# measured with the restatement over frames 0..11 at the default LNI parameters (r = 3, eps = 0.01, weight 0.005): rotation at most
# 0.77 deg and camera centre at most 1.30 mm.  §6q's raw-intensity reference loop at weight 0.01 reaches 0.43 deg and 0.97 mm, depth alone
# 0.99 deg and 1.83 mm: on this scene, whose frames are 160 x 120, LNI beats depth alone but not the raw reference (DESIGN.md §6r)
TINY_LNI_ROT_DEG = 0.85
TINY_LNI_CENTRE_M = 0.0015


def test_dense_tiny_lni_loop():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    ids = list(range(12))
    odo = tl.run_sequence(s, ids, true[0])                            # the default LNI parameters
    st = [f[0] for f in odo.frames]
    assert st[0] == ANCHORED and all(x == 0 for x in st[1:]), st
    assert odo.color_info[0] == (0, 0.0, 0, 0.0) and all(ci[2] > 100 for ci in odo.color_info[1:])
    r, t = tr.pose_errors(np.array([f[1] for f in odo.frames]), true[ids])
    print("tiny LNI odometry: rot deg max %.3f, centre mm max %.3f (raw reference: 0.43 deg, 0.97 mm; depth alone: 0.99 deg, 1.83 mm)" %
          (r.max(), 1e3 * t.max()))
    assert r.max() < TINY_LNI_ROT_DEG and t.max() < TINY_LNI_CENTRE_M, (r, t)


# ---- 4. the golden fixture -------------------------------------------------------------------------------------------------------
def test_golden_fixture_matches_restatement():
    g = np.load(os.path.join(HERE, "golden", "tiny_track_lni.npz"))
    grid = tr.rr.Grid(g["xyz"], g["sdf"], np.zeros(len(g["sdf"])), g["weight"], g["voxel_size"])
    ids, refs = g["ids"].tolist(), g["ref_ids"].tolist()
    L = int(g["num_levels"])
    color = dict(norm_radius=int(g["norm_radius"]), norm_eps=float(g["norm_eps"]))
    fr = tl.track(grid, g["depth"], g["intensity"], ids, g["pose_in"], refs, g["ref_pose"], tuple(g["dcam"]), color=color, num_levels=L,
                  iterations=g["iterations"].tolist())
    for k, f in enumerate(fr):
        for l in range(L):
            assert f.models[l].tobytes() == g[f"model_{l}"][k].tobytes(), (k, l)
            assert f.ref_inten[l].tobytes() == g[f"ref_intensity_{l}"][k].tobytes() and f.inten[l].tobytes() == g[f"intensity_{l}"][k].tobytes()
        assert f.sys.tobytes() == g["sums"][k].tobytes() and f.sys_c.tobytes() == g["color_sums"][k].tobytes()
        assert [f.status, f.iterations, f.correspondences] == g["outcome"][k].tolist()
        assert [f.first[0], f.last[0]] == g["color_rows"][k].tolist()
        assert np.abs(np.array(f.w2c) - g["pose_out"][k]).max() < 1e-12
