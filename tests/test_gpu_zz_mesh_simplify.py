"""GPU tests of the mesh simplification (i3d_simplify_mesh) against the numpy restatement tests/mesh_simplify_ref.py.  Explicitly rounded
double arithmetic, sequential per-cluster sums and integer atomics only: the bar is BYTE-EQUAL vertices, colours and faces, in order,
and equal counts."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MESH = ("vertices", "colors", "faces")


def _engine(scene):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(scene)
    return e


def _mesh_bytes(m):
    return b"".join(m[k].tobytes() for k in MESH)


def _check(e, m_in, cell):
    """simplifies the resident mesh m_in (as downloaded) on the engine and with the restatement; byte-equal, equal counts"""
    import mesh_simplify_ref as msr
    r = msr.simplify(m_in, cell)
    s = e.simplify_mesh(cell)
    for k in MESH:
        assert s[k].shape == r[k].shape and s[k].tobytes() == r[k].tobytes(), (cell, k)
    got = {k: int(getattr(s["info"], k)) for k in msr.INFO_COUNTS}
    assert got == r["info"], (got, r["info"])
    return s


def _check_cells(e, vs, source, lc, mode="", factors=(2, 4), chain=True):
    """for each factor: extract, simplify at factor * vs; then (chain) the last result simplified again at twice the cell"""
    out = []
    for f in factors:
        m = e.extract_mesh(source, lc, mode)
        s = _check(e, m, f * vs)
        assert 0 < len(s["faces"]) < len(m["faces"])
        out.append(s)
        print(source, lc, mode, f, len(m["faces"]), "->", len(s["faces"]), {k: getattr(s["info"], k) for k in ("num_clusters", "num_faces_collapsed",
                                                                                                             "num_faces_duplicate", "num_faces_degenerate")})
    if chain:
        s2 = _check(e, out[-1], 2 * factors[-1] * vs)
        assert len(s2["faces"]) < len(out[-1]["faces"])
    return out


def _gn_params(s):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    return p


def test_tiny_sources_modes_components(tiny_scene):
    s = tiny_scene
    e = _engine(s)
    for _ in range(2):
        e.gn_iteration(_gn_params(s))          # sdf0 and the refined sdf differ
    vs = float(s["voxel_size"])
    for src in ("fused", "refined"):
        for lc in (False, True):
            _check_cells(e, vs, src, lc)
    _check_cells(e, vs, "refined", True, mode="normals")
    e.upsample_grid()                           # after an upsample: half the voxel size
    _check_cells(e, vs / 2, "refined", False, factors=(2, 4, 8))


def test_small_and_c2(small_scene):
    import torch
    from intrinsic3d_b200.scene import config_scene
    e = _engine(small_scene)
    _check_cells(e, float(small_scene["voxel_size"]), "refined", False)
    s = config_scene("c2", device="cuda" if torch.cuda.is_available() else "cpu")
    e = _engine(s)
    _check_cells(e, float(s["voxel_size"]), "refined", True)
    _check_cells(e, float(s["voxel_size"]), "fused", False, factors=(8,), chain=False)


def test_fused_grid():
    import test_gpu_zz_mesh as tgm
    e = tgm._fused_fixture_engine()
    vs = float(e.download_grid()["voxel_size"])
    _check_cells(e, vs, "fused", True)


def test_tiny_cell_is_identity():
    """A sphere in the positive octant (the tiny scene's sphere straddles the origin, where the closest seam vertices are so near that
    half their spacing puts cell coordinates outside int32)."""
    import test_gpu_zz_mesh as tgm
    import test_mesh as tm
    from test_mesh_simplify import min_chebyshev_spacing
    xyz, sdf, w, rgb = tm.grid(tm._sphere((3.3, 2.6, 4.1), 2.2, half=4))
    e = tgm._engine_with(xyz, sdf, sdf, w, rgb, 0.004)
    m = e.extract_mesh("refined", True)
    s = e.simplify_mesh(0.5 * min_chebyshev_spacing(m["vertices"]))
    assert _mesh_bytes(s) == _mesh_bytes(m)
    assert s["info"].num_clusters == len(m["vertices"]) and s["info"].num_faces_collapsed == 0


def test_whole_mesh_cell_gives_empty_mesh(tmp_path):
    import test_gpu_zz_mesh as tgm
    import test_mesh as tm
    from intrinsic3d_b200.mesh import export_meshes, save_ply
    xyz, sdf, w, rgb = tm.grid(tm._sphere((3.3, 2.6, 4.1), 2.2, half=4))
    e = tgm._engine_with(xyz, sdf, sdf, w, rgb, 0.004)
    m = e.extract_mesh("refined")
    assert len(m["faces"]) > 100
    s = _check(e, m, 1.0)
    assert s["vertices"].shape == (0, 3) and s["faces"].shape == (0, 3) and s["info"].num_clusters == 1
    assert e.L.i3d_download_mesh(e.h, None, None, None) == 0
    with pytest.raises(ValueError):
        save_ply(os.devnull, s)
    with pytest.raises(ValueError):
        export_meshes(e, str(tmp_path / "m"), [""], cell_size=1.0)


def test_export_meshes_with_cell_size(tiny_scene, tmp_path):
    from intrinsic3d_b200.mesh import export_meshes, ply_bytes
    e = _engine(tiny_scene)
    vs = float(tiny_scene["voxel_size"])
    paths = export_meshes(e, str(tmp_path / "m"), ["", "normals"], largest_component_only=True, cell_size=3 * vs)
    for path, mode in zip(paths, ("", "normals")):
        e.extract_mesh("refined", True, mode)
        assert open(path, "rb").read() == ply_bytes(e.simplify_mesh(3 * vs))


def test_golden_fixture():
    import test_gpu_zz_mesh as tgm
    g0 = np.load(os.path.join(HERE, "golden", "tiny_mesh.npz"))
    g = np.load(os.path.join(HERE, "golden", "tiny_mesh_simplify.npz"))
    e = tgm._engine_with(g0["xyz"], g0["sdf0"], g0["sdf_refined"], g0["weight"], g0["rgb"], float(g0["voxel_size"]))
    for k, cell in enumerate(g["cells"]):
        if not g["chained"][k]:
            m = e.extract_mesh("refined", True)
            assert m["faces"].tobytes() == g["in_faces"].tobytes()
        s = e.simplify_mesh(float(cell))
        for key in MESH:
            assert s[key].tobytes() == g[f"{k}_{key}"].tobytes(), (k, key)


def test_c3_run_to_run_bit_identical():
    """Full C3 (2 M voxels) and one upsample (16 M): two calls and two engines give byte-identical simplified meshes."""
    import torch
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c3", device="cuda" if torch.cuda.is_available() else "cpu")
    engines = [_engine(s), _engine(s)]
    vs = float(s["voxel_size"])
    for level in range(2):
        for f in (2, 4, 8):
            res = []
            for e in (engines[0], engines[0], engines[1]):
                e.extract_mesh("refined", False)
                res.append(e.simplify_mesh(f * vs))
            assert _mesh_bytes(res[0]) == _mesh_bytes(res[1]) == _mesh_bytes(res[2]), (level, f)
            i = res[0]["info"]
            assert 0 < i.num_faces
            print(level, f, engines[0].n, {k: getattr(i, k) for k in ("num_clusters", "num_faces_collapsed", "num_faces_duplicate",
                                                                       "num_faces_degenerate", "num_faces", "num_vertices")})
        if level == 0:
            for e in engines:
                e.upsample_grid()
            vs /= 2
    for e in engines:
        e.close()


def test_refusals_leave_resident_mesh(tiny_scene):
    from intrinsic3d_b200.ctypes_defs import I3DSimplifyInfo, I3DSimplifyParams
    e = _engine(tiny_scene)
    info = I3DSimplifyInfo()
    assert e.L.i3d_simplify_mesh(e.h, C.byref(I3DSimplifyParams(0.01, 0)), C.byref(info)) != 0
    assert "no mesh" in e.L.i3d_last_error(e.h).decode()
    assert e.L.i3d_simplify_mesh(e.h, None, C.byref(info)) != 0
    m = e.extract_mesh("refined", True)
    s = e.simplify_mesh(2 * float(tiny_scene["voxel_size"]))

    def resident():
        V, F = len(s["vertices"]), len(s["faces"])
        out = dict(vertices=np.empty((V, 3), np.float32), colors=np.empty((V, 3), np.uint8), faces=np.empty((F, 3), np.int32))
        assert e.L.i3d_download_mesh(e.h, out["vertices"].ctypes.data_as(C.POINTER(C.c_float)), out["colors"].ctypes.data_as(C.POINTER(C.c_uint8)),
                                     out["faces"].ctypes.data_as(C.POINTER(C.c_int32))) == 0
        return out

    for bad, msg in ((0.0, "cell_size"), (-1.0, "cell_size"), (float("nan"), "cell_size"), (float("inf"), "cell_size"), (1e-12, "int32")):
        assert e.L.i3d_simplify_mesh(e.h, C.byref(I3DSimplifyParams(bad, 0)), C.byref(info)) != 0, bad
        assert msg in e.L.i3d_last_error(e.h).decode(), (bad, e.L.i3d_last_error(e.h).decode())
        assert _mesh_bytes(resident()) == _mesh_bytes(s), bad
    with pytest.raises(RuntimeError):
        e.simplify_mesh(-1.0)
    assert len(m["faces"]) > len(s["faces"])
    e.upsample_grid()                                      # a new voxel set drops the resident mesh, simplified or not
    assert e.L.i3d_simplify_mesh(e.h, C.byref(I3DSimplifyParams(0.01, 0)), C.byref(info)) != 0
    assert e.L.i3d_download_mesh(e.h, None, None, None) != 0


def test_state_unchanged_by_simplification(tiny_scene):
    """A GN iteration, a render and the next extraction are byte-identical with and without a simplification in between."""
    s = tiny_scene
    out = []
    for simplify in (False, True):
        e = _engine(s)
        e.gn_iteration(_gn_params(s))
        e.extract_mesh("refined", True)
        if simplify:
            e.simplify_mesh(2 * float(s["voxel_size"]))
            e.simplify_mesh(4 * float(s["voxel_size"]))
        info = e.gn_iteration(_gn_params(s))
        r = e.render_keyframes([0, 1])
        m = e.extract_mesh("fused", False)
        out.append((bytes(info)[:type(info).time_add.offset], e.download_state(), r, m))
    assert out[0][0] == out[1][0]
    for k in out[0][1]:
        assert out[0][1][k].tobytes() == out[1][1][k].tobytes(), k
    for k in out[0][2]:
        if k != "stats":
            assert out[0][2][k].tobytes() == out[1][2][k].tobytes(), k
    assert [dict(x) for x in out[0][2]["stats"]] == [dict(x) for x in out[1][2]["stats"]]
    assert _mesh_bytes(out[0][3]) == _mesh_bytes(out[1][3])
