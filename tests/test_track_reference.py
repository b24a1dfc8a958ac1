"""CPU tests of the photometric term against a reference frame's image through its restatement tests/track_reference_ref.py (DESIGN.md
§6q): the model plane's known answer on an affine image, a frame that is its own reference, each case without a model value, the restated
_ref odometry on the dense tiny sequence, and the golden fixture tests/golden/tiny_track_reference.npz."""
import os

import numpy as np

import track_color_ref as tc
import track_ref as tr
import track_reference_ref as trr
from test_odometry import ANCHORED, dense_tiny, run_sequence
from test_track_color import tiny_fused

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32
DCAM = (64, 48, 50.0, 50.0, 31.5, 23.5)
Z = 0.6                                         # the fronto-parallel plane of the synthetic cases


def _affine(W, H, a=0.3, b=0.004, c=-0.003):
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return (a + b * xx + c * yy).astype(f32), (a, b, c)


def _shifted(dx, dy=0.0, dz=0.0):
    """world -> camera of the identity camera moved by (dx, dy, dz)"""
    return np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, -dx, -dy, -dz], np.float64)


def _model(l, ref_pose, pdepth=None, ref_depth=None, max_distance=0.05):
    cams = tr.level_cams(DCAM, l + 1)
    W, H = cams[l]["W"], cams[l]["H"]
    I, abc = _affine(W, H)
    pd = np.full((48, 64), f32(Z), f32) if pdepth is None else pdepth
    rd = np.full((H, W), f32(Z), f32) if ref_depth is None else ref_depth
    m = trr.ref_model(_shifted(0.0).astype(f32), cams[0], cams[l], l, pd, np.asarray(ref_pose, np.float64).astype(f32), I, rd, f32(max_distance))
    return m, cams, abc


# ---- 1. the model plane ----------------------------------------------------------------------------------------------------------------
def test_model_plane_known_answer_on_an_affine_image():
    for l in (0, 1, 2):
        dx = 0.012
        m, cams, (a, b, c) = _model(l, _shifted(dx))
        cam0, cl = cams[0], cams[l]
        H, W = m.shape
        vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        # the model point of prediction pixel (2^l u, 2^l v) on the plane z = Z, seen from the camera moved by dx
        X = (uu * (1 << l) - float(cam0["cx"])) / float(cam0["fx"]) * Z - dx
        Y = (vv * (1 << l) - float(cam0["cy"])) / float(cam0["fy"]) * Z
        x = float(cl["fx"]) * X / Z + float(cl["cx"])
        y = float(cl["fy"]) * Y / Z + float(cl["cy"])
        inside = (x >= 1.001) & (x < W - 2.001) & (y >= 1.001) & (y < H - 2.001)
        outside = (x < 0.999) | (x >= W - 1.999) | (y < 0.999) | (y >= H - 1.999)
        assert inside.sum() > 0.5 * W * H
        assert np.abs(m[inside] - (a + b * x + c * y)[inside]).max() <= 1e-5, l
        assert np.isnan(m[outside]).all() and outside.any(), l


def test_each_failed_test_gives_the_quiet_nan():
    base, _, _ = _model(0, _shifted(0.005))
    v, u = 20, 30
    assert np.isfinite(base[v, u])
    assert base.view(np.uint32)[np.isnan(base)].tolist() == [0x7FC00000] * int(np.isnan(base).sum())
    # no hit: the prediction pixel has no depth
    pd = np.full((48, 64), f32(Z), f32)
    pd[v, u] = 0.0
    m, _, _ = _model(0, _shifted(0.005), pdepth=pd)
    assert np.isnan(m[v, u]) and np.isfinite(m[v, u + 1])
    # behind the reference camera: turned half a revolution about y; it projects to the same pixels, and a max_distance of 10 m keeps the
    # occlusion test (|0.6 - (-0.6)| = 1.2) passing, so x_r2 > 0 alone rejects it
    behind = np.array([-1, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0], np.float64)
    m, _, _ = _model(0, behind, max_distance=10.0)
    assert np.isnan(m).all()
    # out of bounds: the reference moved sideways so far that the pixel leaves [1, W - 2)
    m, _, _ = _model(0, _shifted(-0.45))
    assert np.isnan(m[v, u]) and np.isfinite(m[v, 5])
    # occluded: the reference sees something 6 cm in front of the point at the rounded pixel
    rd = np.full((48, 64), f32(Z), f32)
    ru = int(np.trunc(f32(50.0) * ((f32(u) - f32(31.5)) / f32(50.0) * f32(Z) - f32(0.005)) / f32(Z) + f32(31.5) + f32(0.5)))
    rd[v, ru] = f32(Z - 0.06)
    m, _, _ = _model(0, _shifted(0.005), ref_depth=rd)
    assert np.isnan(m[v, u]) and np.isfinite(m[v, u + 1])
    # invalid reference depth at the rounded pixel; with a max_distance of 10 m, |0 - 0.6| passes, so d > 0 alone rejects it
    rd[v, ru] = 0.0
    m, _, _ = _model(0, _shifted(0.005), ref_depth=rd, max_distance=10.0)
    assert np.isnan(m[v, u]) and np.isfinite(m[v, u + 1])


def test_a_frame_that_is_its_own_reference_has_no_photometric_residual():
    s, dcam, depth, grid, _, inten, _ = tiny_fused()
    true = tr.aa_to_rt(s["poses_true"])
    p, c = tr.params(), trr.color_params()
    for f in (1, 4):
        fr = trr.RefFrame(depth[f], inten[f], true[f], dcam, p, c, depth[f], inten[f], true[f], grid=grid)
        for l in range(p["num_levels"]):
            ok, _, r = tc.photo_rows(fr.Tf(), fr.rt_in, fr.cams[0], fr.cams[l], l, fr.pdepth, fr.pints[l], fr.inten[l], *fr.grads[l],
                                     fr.depth[l], p["max_distance"], c)
            assert ok.sum() > 50 and np.abs(r[ok]).max() <= 1e-5, (f, l, ok.sum(), np.abs(r[ok]).max())


# ---- 2. the _ref odometry loop ------------------------------------------------------------------------------------------------------
# measured with the restatement over frames 0..11, weight 0.01: rotation at most 0.43 deg (depth alone: 0.99 deg), camera centre at most
# 0.97 mm (depth alone: 1.83 mm)
TINY_REF_ROT_DEG = 0.5
TINY_CENTRE_M = 0.0018


def test_dense_tiny_reference_loop_beats_depth_only():
    s = dense_tiny(72)
    true = tr.aa_to_rt(s["poses_true"])
    ids = list(range(12))
    odo = trr.run_sequence(s, ids, true[0])                          # the default weight, 0.01
    st = [f[0] for f in odo.frames]
    assert st[0] == ANCHORED and all(x == 0 for x in st[1:]), st
    assert odo.color_info[0] == (0, 0.0, 0, 0.0) and all(ci[2] > 100 for ci in odo.color_info[1:])
    r, t = tr.pose_errors(np.array([f[1] for f in odo.frames]), true[ids])
    geo = run_sequence(s, ids, true[0])
    rg, _ = tr.pose_errors(np.array([f[1] for f in geo.frames]), true[ids])
    print("tiny reference odometry: rot deg max %.3f (depth only %.3f), centre mm max %.3f" % (r.max(), rg.max(), 1e3 * t.max()))
    assert r.max() < rg.max(), (r.max(), rg.max())
    assert r.max() < TINY_REF_ROT_DEG and t.max() < TINY_CENTRE_M, (r, t)


# ---- 3. the golden fixture -------------------------------------------------------------------------------------------------------
def test_golden_fixture_matches_restatement():
    g = np.load(os.path.join(HERE, "golden", "tiny_track_reference.npz"))
    grid = tr.rr.Grid(g["xyz"], g["sdf"], np.zeros(len(g["sdf"])), g["weight"], g["voxel_size"])
    ids, refs = g["ids"].tolist(), g["ref_ids"].tolist()
    L = int(g["num_levels"])
    fr = trr.track(grid, g["depth"], g["intensity"], ids, g["pose_in"], refs, g["ref_pose"], tuple(g["dcam"]), num_levels=L,
                   iterations=g["iterations"].tolist())
    for k, f in enumerate(fr):
        for l in range(L):
            assert f.models[l].tobytes() == g[f"model_{l}"][k].tobytes(), (k, l)
            assert f.ref_inten[l].tobytes() == g[f"ref_intensity_{l}"][k].tobytes() and f.ref_depth[l].tobytes() == g[f"ref_depth_{l}"][k].tobytes()
        assert f.sys.tobytes() == g["sums"][k].tobytes() and f.sys_c.tobytes() == g["color_sums"][k].tobytes()
        assert [f.status, f.iterations, f.correspondences] == g["outcome"][k].tolist()
        assert [f.first[0], f.last[0]] == g["color_rows"][k].tolist()
        assert np.abs(np.array(f.w2c) - g["pose_out"][k]).max() < 1e-12
