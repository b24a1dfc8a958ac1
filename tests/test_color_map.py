"""CPU tests of the colour map optimisation restatement (tests/color_map_ref.py, DESIGN.md §6y): the samples, the Jacobian against
float64 finite differences, the solve's exclusions and fixed keyframes, and the measured behaviour on the tiny scene that kept the
method from being built on the device."""
import math

import numpy as np
import pytest

import color_map_ref as cm
import distance_ref
import texture_ref
import track_ref

f32 = np.float32


def _tiny():
    import mesh_ref
    import render_ref as rr
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("tiny")
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], s["rgb"], float(s["voxel_size"]), False)
    return s, m, rr.camera(s["intr"], s["dist"]), cm.pose_rt64(s["poses_true"])


@pytest.mark.parametrize("L", [1, 2, 3])
def test_samples_are_the_distance_samples_with_the_bake_normals(L):
    rng = np.random.default_rng(L)
    V = rng.standard_normal((40, 3)).astype(f32)
    faces = np.array([rng.choice(40, 3, replace=False) for _ in range(60)])
    faces[5] = (3, 3, 7)                                                # a degenerate face: zero normal, its samples dropped
    mesh = dict(vertices=V, faces=faces)
    P, N, valid = cm.samples(mesh, L)
    Pd, _ = distance_ref.samples(mesh, L)
    assert P.tobytes() == Pd.tobytes() and len(P) == 60 * L * L
    n = texture_ref.face_normals(V, faces.astype(np.int64))
    assert N.tobytes() == np.repeat(n, L * L, axis=0).tobytes()
    assert not valid[5 * L * L:6 * L * L].any() and valid.sum() == 59 * L * L


@pytest.mark.parametrize("dist", [(0.0, 0.0, 0.0, 0.0, 0.0), (-0.12, 0.05, -0.01, 0.004, -0.003)])
def test_jacobian_matches_finite_differences(dist):
    """On a linear image the bilinear value and the central differences are exact, so the float64 row must equal the derivative of the
    float64 residual under T <- [Rodrigues(w) | v] T; the float32 row must agree with it to float rounding."""
    W, H = 400, 300
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    lum = 0.3 + 0.0021 * u - 0.0013 * v
    cam = dict(fx=f32(280.0), fy=f32(275.0), cx=f32(199.5), cy=f32(149.5), d=np.array(dist, f32))
    rng = np.random.default_rng(3)
    T = np.array(track_ref.update([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], [0.1, -0.05, 0.02, 0.01, -0.02, 0.3]))
    R, t = T[:9].reshape(3, 3), T[9:]
    qc = np.stack([rng.uniform(-0.25, 0.25, 500), rng.uniform(-0.2, 0.2, 500), rng.uniform(0.8, 1.3, 500)], 1)
    P = (qc - t) @ R                                                    # world points whose camera points are qc
    q = [P @ R[k] + t[k] for k in range(3)]
    _, _, _, _, pu, pv = cm.project(q, cam, np.float64)
    inside, _, gu, gv = cm.sample_image(lum, pu, pv, np.float64)
    assert inside.all()
    J = cm.row(q, gu, gv, cam, np.float64)
    h = 1e-6
    Jn = np.zeros_like(J)
    for a in range(6):
        x = [0.0] * 6
        x[a] = h
        rp = cm.residual(P, track_ref.update(list(T), x), cam, lum, 0.0)
        x[a] = -h
        rm = cm.residual(P, track_ref.update(list(T), x), cam, lum, 0.0)
        Jn[:, a] = (rp - rm) / (2 * h)
    scale = np.abs(Jn).max(0)
    assert np.all(np.abs(J - Jn).max(0) <= 1e-6 * scale), np.abs(J - Jn).max(0) / scale
    q32 = [a.astype(f32) for a in q]
    J32 = cm.row(q32, gu.astype(f32), gv.astype(f32), cam)
    assert J32.dtype == f32 and np.all(np.abs(J32 - J).max(0) <= 1e-4 * scale)


def test_colours_are_the_weighted_mean_and_respect_min_views():
    s, m, cam, Tt = _tiny()
    prob = cm.Problem(m, s["lum"], s["depth"], cam, 1, 0.02)
    C, views, Wt, It = prob.colours(Tt, 2)
    used = views >= 2
    assert used.sum() > 0.5 * len(C) and np.isnan(C[~used]).all()
    ref = (Wt.astype(np.float64) * It).sum(1)[used] / Wt.astype(np.float64).sum(1)[used]
    assert np.array_equal(C[used], ref.astype(f32))
    C3, views3, _, _ = prob.colours(Tt, 3)
    assert np.array_equal(views3, views) and np.array_equal(~np.isnan(C3), views >= 3)


def test_fixed_keyframes_and_exclusions():
    s, m, cam, Tt = _tiny()
    F = len(Tt)
    prob = cm.Problem(m, s["lum"], s["depth"], cam, 1, 0.02)
    T0 = track_ref.perturb(Tt, 0.3, 0.003, 3)
    fixed = np.zeros(F, bool)
    fixed[[0, 2]] = True
    T, st, info, _, _ = cm.optimize(prob, T0, fixed, iterations=2)
    assert T[0].tobytes() == T0[0].tobytes() and T[2].tobytes() == T0[2].tobytes()
    assert st[0] == cm.FIXED and st[2] == cm.FIXED and np.all(st[~fixed] == cm.OK)
    assert not np.array_equal(T[~fixed], T0[~fixed])
    # no sample reaches min_views: no rows, every free keyframe too few rows, nothing moves
    T, st, info, C, sys_ = cm.optimize(prob, T0, fixed, iterations=2, min_views=F + 1)
    assert np.isnan(C).all() and info["samples_used"] == 0 and info["rows"] == 0
    assert np.all(st[~fixed] == cm.FEW_ROWS) and T.tobytes() == T0.tobytes()
    # min_rows above every keyframe's row count
    T, st, info, _, sys_ = cm.optimize(prob, T0, fixed, iterations=2, min_rows=10 ** 6)
    assert np.all(st[~fixed] == cm.FEW_ROWS) and T.tobytes() == T0.tobytes() and info["iterations"] == 1
    # a singular system: a keyframe whose rows all have zero gradient
    S = np.zeros(cm.VALS)
    S[28] = 100
    assert cm.solve(S, 1e-4)[0] == cm.NOT_PD
    S[3] = np.inf
    assert cm.solve(S, 1e-4)[0] == cm.NON_FINITE


# Measured on the tiny scene (refined mesh, L = 1, the default parameters, 30 iterations), DESIGN.md §6y: keyframes 1-5 perturbed by
# 0.3 deg / 3 mm (track_ref.perturb, seed 3), keyframe 0 fixed at the truth.  The energy falls from 5.72 to 4.50 while the rotation
# errors grow to 1.8-4.9 deg; the energy at the true poses is 4.00.  The Gauss-Newton alternation finds a lower-energy state than its
# start but not the truth, so the method was not built on the device.
def test_measured_alternation_on_tiny_moves_away_from_the_truth():
    s, m, cam, Tt = _tiny()
    F = len(Tt)
    prob = cm.Problem(m, s["lum"], s["depth"], cam, 1, 0.02)
    T0 = track_ref.perturb(Tt, 0.3, 0.003, 3)
    T0[0] = Tt[0]
    fixed = np.zeros(F, bool)
    fixed[0] = True
    T, st, info, _, _ = cm.optimize(prob, T0, fixed)
    rot0, _ = track_ref.pose_errors(T0, Tt)
    rot1, _ = track_ref.pose_errors(T, Tt)
    _, _, truth, _, _ = cm.optimize(prob, Tt, np.ones(F, bool), iterations=0)
    print("rotation error (deg) before", np.round(rot0, 3).tolist(), "after", np.round(rot1, 3).tolist(),
          "energy %.3f -> %.3f, at the truth %.3f" % (info["energy_before"], info["energy_after"], truth["energy_after"]))
    assert info["energy_after"] < info["energy_before"]
    assert truth["energy_after"] < info["energy_after"]
    assert rot1[1:].min() > 1.0 > 0.35 > rot0[1:].max()
