"""CPU tests of the reference-mesh registration restatement tests/register_ref.py (DESIGN.md §6aa): the row against central differences,
exact-copy recovery, the statuses of degenerate problems, the normal gate, the transform rule and the fixture."""
import math
import os

import numpy as np
import pytest

import grid_from_mesh_ref as gr
import register_ref as rg

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32


@pytest.fixture(scope="module")
def tiny_sdf0():
    import mesh_ref
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("tiny")
    vs = float(s["voxel_size"])
    return mesh_ref.extract(s["xyz"], s["sdf0"], s["weight"], s["rgb"], vs, True), vs


def _residual(xi, p, c, n):
    """float64 point-to-plane residual of p moved by [Rodrigues(w) | v], xi = (w, v)"""
    R = np.array(rg.tr.rodrigues(list(xi[:3]))).reshape(3, 3)
    return float(n @ (R @ p + xi[3:] - c))


def test_row_against_central_differences(tiny_sdf0):
    A, vs = tiny_sdf0
    B = rg.moved(A, rg.motion(1.0, 0.5 * vs, 3))
    R = rg.rows(A, B, rg.tr.inverse(rg.IDENTITY), 1, f32(0.016), f32(0.5))
    k = np.flatnonzero(R["kept"])
    assert len(k) > 0.9 * len(R["kept"])
    nB = rg.face_normals(B)
    v = np.asarray(B["vertices"], np.float64)
    f = np.asarray(B["faces"])
    h = 1e-6
    for i in k[:: max(1, len(k) // 50)]:
        p = R["p"][i].astype(np.float64)
        n = nB[R["face"][i]].astype(np.float64)
        c = p - R["r"][i] * n                   # a point on the plane of the face
        assert abs(n @ (c - v[f[R["face"][i], 0]])) <= 1e-6
        for j in range(6):
            e = np.zeros(6); e[j] = h
            d = (_residual(e, p, c, n) - _residual(-e, p, c, n)) / (2 * h)
            assert abs(d - R["J"][i, j]) <= 1e-7, (i, j, d, R["J"][i, j])
        assert abs(_residual(np.zeros(6), p, c, n) - R["r"][i]) <= 1e-9


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_exact_copy_recovered(tiny_sdf0, seed):
    A, vs = tiny_sdf0
    G = rg.motion(3.0, 2 * vs, seed, np.asarray(A["vertices"], np.float64).mean(0))
    B = rg.moved(A, G)
    out = rg.register(A, B)
    assert out["status"] == 0 and out["iterations"] == 30
    rot, disp = rg.errors(out["T"], rg.tr.inverse(list(G)), B["vertices"])
    assert rot <= 1e-3 and disp <= 1e-3 * vs, (rot, disp / vs)
    n0, w0, _, rms0 = rg.summary(out["systems"][0])
    n1, w1, _, rms1 = rg.summary(out["systems"][-1])
    assert n1 == len(A["faces"]) and rms1 < 1e-3 * rms0


def test_parallel_squares_not_positive_definite():
    A = gr.square_patch(-0.02, 0.02, 0.0, n=4)
    B = gr.square_patch(-0.02, 0.02, 0.001, n=6)
    out = rg.register(A, B, min_correspondences=6)
    assert out["status"] == 2 and out["iterations"] == 0
    S = out["systems"][0]
    assert int(S[28]) == len(A["faces"])
    # the w_z, v_x and v_y columns are exactly zero
    for j, (a, b) in enumerate(rg.tr.UPPER):
        if a in (2, 3, 4) or b in (2, 3, 4):
            assert S[j] == 0.0
    np.testing.assert_array_equal(out["T"], rg.IDENTITY)


def test_too_far_few_correspondences():
    A = gr.square_patch(-0.02, 0.02, 0.0, n=4)
    B = gr.square_patch(-0.02, 0.02, 0.05, n=4)
    out = rg.register(A, B, min_correspondences=6)
    assert out["status"] == 1 and out["iterations"] == 0 and int(out["systems"][0][28]) == 0


def test_normal_gate_on_thin_slab():
    th = 0.0005
    B = gr.box_mesh([-0.02, -0.02, 0.0], [0.02, 0.02, th])
    A = gr.square_patch(-0.015, 0.015, 0.3 * th, n=4)         # normal +z, nearer the slab's bottom (normal -z) than its top
    assert rg.face_normals(A)[:, 2].min() == 1.0
    M = rg.tr.inverse(rg.IDENTITY)
    gated = rg.rows(A, B, M, 2, f32(0.004), f32(0.5))
    open_ = rg.rows(A, B, M, 2, f32(0.004), f32(-1.0))
    assert (open_["face"] >= 0).all() and open_["kept"].all()
    assert not gated["kept"].any()
    # with the top of the slab nearer, the gate keeps every sample
    A2 = gr.square_patch(-0.015, 0.015, 0.7 * th, n=4)
    assert rg.rows(A2, B, M, 2, f32(0.004), f32(0.5))["kept"].all()


def test_transform_rule():
    rng = np.random.default_rng(4)
    v = rng.normal(0, 0.1, (500, 3)).astype(f32)
    np.testing.assert_array_equal(rg.transform(v, rg.IDENTITY), v)
    G = rg.motion(7.0, 0.03, 5)
    out = rg.transform(v, G)
    ref = v.astype(np.float64) @ G[:9].reshape(3, 3).T + G[9:]
    assert np.abs(out - ref).max() <= 2 * np.spacing(np.abs(ref).max().astype(f32))
    # x <- G^-1 (G x) comes back to within float rounding
    back = rg.transform(out, rg.tr.inverse(list(G)))
    assert np.abs(back - v).max() <= 1e-7


def test_fixture():
    z = np.load(os.path.join(HERE, "golden", "tiny_register.npz"))
    A = dict(vertices=z["a_vertices"], faces=z["a_faces"])
    B = dict(vertices=z["b_vertices"], faces=z["a_faces"])
    out = rg.register(A, B, max_distance=(0.016, 0.008), iterations=(3, 3))
    assert out["status"] == int(z["status"]) and out["iterations"] == int(z["iterations"])
    np.testing.assert_array_equal(out["systems"], z["systems"])
    np.testing.assert_array_equal(out["Ms"], z["poses"])
    np.testing.assert_array_equal(out["T"], z["T"])
    f0 = rg.rows(A, B, rg.tr.inverse(rg.IDENTITY), 1, f32(0.016), f32(0.5))["face"]
    np.testing.assert_array_equal(f0, z["faces0"])
    rot, disp = rg.errors(out["T"], rg.tr.inverse(list(z["G"])), B["vertices"])
    assert rot < 1e-3 and disp < 1e-5 and math.isfinite(out["update_norm"])
