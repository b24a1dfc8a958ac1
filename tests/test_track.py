"""CPU tests of the tracking restatement tests/track_ref.py (DESIGN.md §6n): the analytic Jacobian, an analytically constructed corner, the
tiny scene's tracking accuracy, and the golden fixture tests/golden/tiny_track.npz."""
import math
import os

import numpy as np
import pytest

import render_ref as rr
import track_ref as tr

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32


def _residual(xi, p, q, n):
    """n . (Rodrigues(w) p + v - q) in float64"""
    R = np.array(tr.rodrigues(list(xi[:3]))).reshape(3, 3)
    return n @ (R @ p + xi[3:] - q)


def test_kt1_jacobian_matches_central_differences():
    rng = np.random.default_rng(11)
    for _ in range(50):
        p = rng.normal(size=3).astype(f32)
        q = (p + 0.01 * rng.normal(size=3)).astype(f32)
        n = rng.normal(size=3); n = (n / np.linalg.norm(n)).astype(f32)
        ok = np.ones((1, 1), bool)
        J, r = tr.rows(ok, [np.full((1, 1), p[k]) for k in range(3)], [np.full((1, 1), q[k]) for k in range(3)],
                       [np.full((1, 1), n[k]) for k in range(3)])
        pd, qd, nd = p.astype(np.float64), q.astype(np.float64), n.astype(np.float64)
        assert r[0, 0] == pytest.approx(_residual(np.zeros(6), pd, qd, nd), rel=1e-12, abs=1e-15)
        h = 1e-6
        num = np.array([(_residual(h * e, pd, qd, nd) - _residual(-h * e, pd, qd, nd)) / (2 * h) for e in np.eye(6)])
        assert np.allclose(J[0, 0], num, rtol=1e-6, atol=1e-8), (J[0, 0], num)


def _look_at(c, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """world -> camera R | t [12] of a camera at c looking at target"""
    c = np.asarray(c, np.float64)
    z = np.asarray(target, np.float64) - c; z /= np.linalg.norm(z)
    x = np.cross(z, up); x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return np.concatenate([R.reshape(-1), -R @ c])


def _planes_view(rt, dcam, planes):
    """analytic depth and world normals of the axis planes k in `planes` (x_k = 0, bounding the octant x, y, z >= 0 where the camera is)
    seen from rt: the first plane a ray leaves the octant through"""
    W, H, fx, fy, cx, cy = dcam
    R, t = np.asarray(rt[:9], np.float64).reshape(3, 3), np.asarray(rt[9:], np.float64)
    o = -R.T @ t
    vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    d = np.stack([(uu - cx) / fx, (vv - cy) / fy, np.ones_like(uu, dtype=np.float64)], -1) @ R        # R^T (x, y, 1): camera z = 1
    depth = np.full((H, W), np.inf)
    nrm = np.zeros((H, W, 3))
    for k in planes:
        with np.errstate(divide="ignore", invalid="ignore"):
            s = -o[k] / d[..., k]
        hit = o[None, None, :] + s[..., None] * d
        inside = np.all(np.delete(hit, k, axis=-1) >= 0, -1) if len(planes) > 1 else np.ones_like(s, bool)
        better = (d[..., k] < 0) & (s > 0) & inside & (s < depth)
        depth = np.where(better, s, depth)
        nrm[better] = np.eye(3)[k]
    depth[~np.isfinite(depth)] = 0
    return depth.astype(f32), nrm.astype(f32)


DCAM = (64, 48, 50.0, 50.0, 31.5, 23.5)


def _corner_frame(planes, delta, **over):
    true = _look_at((0.6, 0.5, 0.7))
    c_in = np.array([0.6, 0.5, 0.7]) + delta
    R = true[:9].reshape(3, 3)
    pose_in = np.concatenate([true[:9], -R @ c_in])
    depth, _ = _planes_view(true, DCAM, planes)
    pred = _planes_view(pose_in.astype(f32).astype(np.float64), DCAM, planes)
    p = tr.params(num_levels=1, iterations=(1,), **over)
    return tr.Frame(depth, pose_in, DCAM, p, prediction=pred).run(), true


def test_kt2_corner_translation_in_one_iteration():
    fr, true = _corner_frame((0, 1, 2), np.array([0.004, -0.003, 0.002]))
    assert fr.status == 0 and fr.iterations == 1 and fr.correspondences > 1500
    rot, trans = tr.pose_errors([fr.w2c], [true])
    assert rot[0] < 1e-4 and trans[0] < 2e-6, (rot, trans)           # 5 mm recovered to float rounding of the planes
    # the solved rotation is zero to rounding: the rows of three orthogonal planes are linear in the translation
    assert np.abs(np.array(fr.T[:9]) - true[:9].reshape(3, 3).T.reshape(-1)).max() < 1e-6


def test_kt2_single_plane_is_not_positive_definite():
    fr, _ = _corner_frame((2,), np.array([0.004, -0.003, 0.002]))
    assert fr.status == 2 and fr.iterations == 0 and fr.correspondences > 1500


def test_kt2_too_few_correspondences_freeze():
    fr, _ = _corner_frame((0, 1, 2), np.array([0.004, -0.003, 0.002]), min_correspondences=100000)
    assert fr.status == 1 and fr.iterations == 0


# The achieved errors of the tiny scene (sdf0 with 0.1-voxel noise, a bumpy sphere of 4 cm radius at 160 x 120), measured with the
# restatement (DESIGN.md §6n): translation errors end >= 10x below the start; rotation about the sphere's centre is constrained only by
# its 3 % bumps, so rotation errors end at 0.09-0.63 degrees whatever the start, and that measured bound is the gate.
KT3_ROT_DEG = 0.7
KT3_TRANS_M_SCENE = 6e-4
KT3_TRANS_RATIO_PERTURBED = 10.0


def kt3_cases(s):
    true = tr.aa_to_rt(s["poses_true"])
    return true, {"scene": tr.aa_to_rt(s["poses"]), "1cm_1deg": tr.perturb(true, 1.0, 0.01, seed=5)}


def check_kt3(name, start, out, true):
    r0, t0 = tr.pose_errors(start, true)
    r1, t1 = tr.pose_errors(out, true)
    assert (r1 < KT3_ROT_DEG).all(), (name, r0, r1)
    if name == "scene":
        assert (t1 < KT3_TRANS_M_SCENE).all(), (name, t0, t1)
    else:
        assert (t1 * KT3_TRANS_RATIO_PERTURBED <= t0).all() and (r1 < r0).all(), (name, r0, r1, t0, t1)
    return r1, t1


def test_kt3_tiny_scene_accuracy(tiny_scene):
    s = tiny_scene
    g = rr.Grid(s["xyz"], s["sdf0"], s["albedo"], s["weight"], s["voxel_size"])
    F, H, W = s["depth"].shape
    dcam = (W, H) + tuple(float(v) for v in s["intr"])
    true, cases = kt3_cases(s)
    for name, start in cases.items():
        fr = tr.track(g, s["depth"], list(range(F)), start, dcam)
        assert all(f.status == 0 and f.iterations == 19 for f in fr)
        check_kt3(name, start, np.array([f.w2c for f in fr]), true)


def test_golden_fixture_matches_restatement():
    g = np.load(os.path.join(HERE, "golden", "tiny_track.npz"))
    grid = rr.Grid(g["xyz"], g["sdf0"], g["albedo"], g["weight"], g["voxel_size"])
    ids = g["ids"].tolist()
    fr = tr.track(grid, g["depth"], ids, g["pose_in"], tuple(g["dcam"]), num_levels=int(g["num_levels"]), iterations=g["iterations"].tolist())
    for k, f in enumerate(fr):
        for l in range(int(g["num_levels"])):
            assert f.depth[l].tobytes() == g[f"depth_{l}"][k].tobytes()
            assert f.nrm[l].tobytes() == g[f"normal_{l}"][k].tobytes()
        assert f.pdepth.tobytes() == g["pred_depth"][k].tobytes() and f.pnrm.tobytes() == g["pred_normal"][k].tobytes()
        assert f.mask.tobytes() == g["mask"][k].tobytes()
        assert f.sys.tobytes() == g["sums"][k].tobytes()
        assert [f.status, f.iterations, f.correspondences] == g["outcome"][k].tolist()
        assert np.abs(np.array(f.w2c) - g["pose_out"][k]).max() < 1e-12
