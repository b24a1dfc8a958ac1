"""GPU tests of the reference-mesh registration (i3d_register_reference_mesh, i3d_transform_reference_mesh) against the numpy restatement
tests/register_ref.py.  Every system is checked with the restatement driven by the device's own pose for it: the sums to 1e-12, the poses
after each update to 1e-12, the per-sample faces at the initial pose byte-equal.  Also known answers, identity, isolation and the fixture."""
import os

import numpy as np
import pytest

import register_ref as rg

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32
SHORT = dict(max_distance=(0.016, 0.008, 0.004), iterations=(3, 2, 2))


def _engine(s):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(s)
    return e


def _truth(name):
    from intrinsic3d_b200.scene import config_geometry, truth_mesh
    return truth_mesh(**config_geometry(name))


def _check_systems(e, A, B, L, sched, T_init=None):
    """the device's systems, poses and first faces against the restatement driven by the device's poses"""
    T, info = e.register_reference_mesh(samples_per_edge=L, init=T_init, **sched)
    S, M, faces = e.debug_register_systems(len(A["faces"]) * L * L)
    r = rg.register(A, B, T_init=T_init, poses=M, samples_per_edge=L, **sched)
    assert S.shape == r["systems"].shape
    for k in range(len(S)):
        scale = np.abs(r["systems"][k][:29]).max()
        assert np.abs(S[k][:29] - r["systems"][k][:29]).max() <= 1e-12 * max(scale, 1e-300), k
    for k in (0, len(S) - 1):
        np.testing.assert_allclose(S[k][29], r["systems"][k][29], rtol=1e-12, atol=0)
    # the pose after each applied update, from the device's pose before it
    for k in range(len(S) - 1):
        if not np.array_equal(M[k], M[k + 1]):
            st, x = rg.tr.solve(S[k][:29])
            assert st == 0
            np.testing.assert_allclose(M[k + 1], rg.tr.update(list(M[k]), x), rtol=0, atol=1e-12)
    f0 = rg.rows(A, B, M[0], L, f32(sched["max_distance"][0]), f32(0.5))["face"]
    assert faces.tobytes() == f0.tobytes()
    assert info.status == r["status"] and info.iterations == r["iterations"]
    np.testing.assert_allclose(T, rg.tr.inverse(list(M[-1])), rtol=0, atol=1e-12)
    n0, w0, sq0, _ = rg.summary(S[0])
    assert (info.initial_rows, info.final_rows) == (n0, int(S[-1][28]))
    assert info.initial_weight == w0 and info.initial_residual_sq == sq0
    return T, info


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_against_restatement(name, tiny_scene, small_scene):
    s = tiny_scene if name == "tiny" else small_scene
    vs = float(s["voxel_size"])
    e = _engine(s)
    truth = _truth(name)
    e.upload_reference_mesh(truth)
    for simplified in (False, True):
        A = e.extract_mesh("fused", False)
        if simplified:
            A = e.simplify_mesh(2 * vs)
        for L in (1, 2):
            _check_systems(e, A, truth, L, SHORT)
    # from a perturbed start, on a moved copy
    A = e.extract_mesh("fused", False)
    G = rg.motion(2.0, vs, 5, np.asarray(A["vertices"], np.float64).mean(0))
    B = rg.moved(A, G)
    e.upload_reference_mesh(B)
    _check_systems(e, A, B, 1, SHORT, T_init=rg.motion(0.5, 0.3 * vs, 6))


def test_known_answers(tiny_scene):
    s = tiny_scene
    vs = float(s["voxel_size"])
    e = _engine(s)
    A = e.extract_mesh("fused", True)
    for seed in range(3):
        G = rg.motion(3.0, 2 * vs, seed, np.asarray(A["vertices"], np.float64).mean(0))
        B = rg.moved(A, G)
        e.upload_reference_mesh(B)
        T, info = e.register_reference_mesh()
        assert info.status == 0 and info.iterations == 30
        rot, disp = rg.errors(T, rg.tr.inverse(list(G)), B["vertices"])
        assert rot <= 1e-3 and disp <= 1e-3 * vs, (rot, disp / vs)
        e.transform_reference_mesh(T)
        assert e.surface_distance((0.1 * vs,), 2 * vs, 2)["accuracy"]["mean"] <= 1e-3 * vs
    # the truth registered against the sdf0 mesh: close to the identity, as the restatement finds it
    truth = _truth("tiny")
    e.upload_reference_mesh(truth)
    T, info = e.register_reference_mesh()
    r = rg.register(A, truth)
    assert info.status == r["status"] == 0
    # two independent trajectories: a last-bit difference of the update (sin, cos) can flip a rounding of the float pose
    np.testing.assert_allclose(T, r["T"], rtol=0, atol=1e-6)
    rot, disp = rg.errors(T, rg.IDENTITY, truth["vertices"])
    rr, rd = rg.errors(r["T"], rg.IDENTITY, truth["vertices"])
    # measured by the restatement: 0.136 degrees (the sphere's rotation is held by its bumps only) and 0.026 voxel
    assert abs(rot - rr) <= 1e-4 and abs(disp - rd) <= 1e-4 * vs and rot < 0.2 and disp < 0.05 * vs


def test_identity_cells_and_engines(small_scene):
    s = small_scene
    vs = float(s["voxel_size"])
    out = []
    for _ in range(2):
        e = _engine(s)
        e.extract_mesh("fused", False)
        e.upload_reference_mesh(_truth("small"))
        for cell in (None, None, 1.5 * vs, 6 * vs):
            T, info = e.register_reference_mesh(cell_size=cell)
            S, M, f = e.debug_register_systems(int(info.num_samples))
            out.append((T.tobytes(), S.tobytes(), M.tobytes(), f.tobytes(), info.status, info.iterations, info.final_rms))
        e.close()
    assert all(o == out[0] for o in out)


def test_refusals_change_nothing(tiny_scene):
    s = tiny_scene
    vs = float(s["voxel_size"])
    e = _engine(s)
    with pytest.raises(RuntimeError, match="no mesh"):
        e.register_reference_mesh()
    A = e.extract_mesh("fused", False)
    with pytest.raises(RuntimeError, match="no reference"):
        e.register_reference_mesh()
    with pytest.raises(RuntimeError, match="no reference"):
        e.transform_reference_mesh(rg.IDENTITY)
    e.upload_reference_mesh(_truth("tiny"))
    before = e.surface_distance((0.1 * vs,), 2 * vs, 2)
    vd0, vf0 = before["vertex_distance"].copy(), before["vertex_face"].copy()
    bad_T = [np.full(12, np.nan), np.r_[2 * np.eye(3).ravel(), 0, 0, 0], np.r_[np.diag([1.0, 1.0, -1.0]).ravel(), 0, 0, 0]]
    bad = [dict(samples_per_edge=0), dict(samples_per_edge=17), dict(max_distance=(0.004, 0.008), iterations=(1, 1)),
           dict(max_distance=(np.inf,), iterations=(1,)), dict(max_distance=(0.0,), iterations=(1,)), dict(max_distance=(0.01,), iterations=(-1,)),
           dict(max_distance=(0.01, 0.01), iterations=(200, 57)), dict(min_normal_cos=1.5), dict(min_correspondences=5),
           dict(cell_size=-1.0), dict(cell_size=1e-6)] + [dict(init=T) for T in bad_T]
    for kw in bad:
        with pytest.raises(RuntimeError):
            e.register_reference_mesh(**kw)
    for T in bad_T:
        with pytest.raises(RuntimeError):
            e.transform_reference_mesh(T)
    import ctypes as C
    assert e.L.i3d_register_reference_mesh(e.h, None, None, None, None) != 0
    vd, vf = np.empty_like(vd0), np.empty_like(vf0)
    e._check(e.L.i3d_download_surface_distance(e.h, vd.ctypes.data_as(C.POINTER(C.c_float)), vf.ctypes.data_as(C.POINTER(C.c_int32))))
    assert vd.tobytes() == vd0.tobytes() and vf.tobytes() == vf0.tobytes()
    after = e.surface_distance((0.1 * vs,), 2 * vs, 2)
    for side in ("accuracy", "completeness"):
        assert {k: v for k, v in after[side].items() if not k.startswith("ms_")} == {k: v for k, v in before[side].items() if not k.startswith("ms_")}
    # a successful registration keeps them too
    e.register_reference_mesh()
    e._check(e.L.i3d_download_surface_distance(e.h, vd.ctypes.data_as(C.POINTER(C.c_float)), vf.ctypes.data_as(C.POINTER(C.c_int32))))
    assert vd.tobytes() == vd0.tobytes() and vf.tobytes() == vf0.tobytes()
    m = e._download_mesh(A["info"])
    assert m["vertices"].tobytes() == A["vertices"].tobytes() and m["faces"].tobytes() == A["faces"].tobytes()


def test_other_results_unchanged(tiny_scene):
    """A GN iteration, an extraction, a render and a bake are byte-identical with and without registration calls"""
    from intrinsic3d_b200.ctypes_defs import default_params
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    outs = []
    for reg in (False, True):
        e = _engine(s)
        e.upload_color_frames(col)
        e.extract_mesh("fused", False)
        e.upload_reference_mesh(_truth("tiny"))
        if reg:
            e.register_reference_mesh()
        it = e.gn_iteration(p)
        m = e.extract_mesh("refined", True)
        if reg:
            e.register_reference_mesh()
        r = e.render_keyframes([0, 2])
        t = e.bake_texture(8)
        outs.append((it.cost_initial, it.cost_final, e.download_state()["sdf_refined"].tobytes(), m["vertices"].tobytes(), m["faces"].tobytes(),
                     r["depth"].tobytes(), r["normal"].tobytes(), t["image"].tobytes(), t["uv"].tobytes()))
        e.close()
    assert outs[0] == outs[1]


def test_fixture_on_device(tiny_scene):
    z = np.load(os.path.join(HERE, "golden", "tiny_register.npz"))
    e = _engine(tiny_scene)
    A = e.extract_mesh("fused", True)
    assert A["vertices"].tobytes() == z["a_vertices"].tobytes() and A["faces"].tobytes() == z["a_faces"].tobytes()
    e.upload_reference_mesh(dict(vertices=z["b_vertices"], faces=z["a_faces"]))
    T, info = e.register_reference_mesh(max_distance=(0.016, 0.008), iterations=(3, 3))
    S, M, f = e.debug_register_systems(len(z["a_faces"]))
    assert f.tobytes() == z["faces0"].tobytes()
    assert info.status == int(z["status"]) and info.iterations == int(z["iterations"])
    # the first system is formed at the identity on both sides; the later ones follow two independent trajectories
    assert np.abs(S[0][:29] - z["systems"][0][:29]).max() <= 1e-12 * np.abs(z["systems"][0][:29]).max()
    np.testing.assert_allclose(M, z["poses"], rtol=0, atol=1e-8)
    for k in range(1, len(S)):
        assert np.abs(S[k][:29] - z["systems"][k][:29]).max() <= 1e-5 * np.abs(z["systems"][k][:29]).max()
    np.testing.assert_allclose(T, z["T"], rtol=0, atol=1e-8)
