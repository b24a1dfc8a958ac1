"""GPU tests of the surface extraction (i3d_extract_mesh / i3d_download_mesh) against the numpy restatement tests/mesh_ref.py.
Exact-rounding float work, integer welding and integer atomics: the bar is BYTE-EQUAL vertices, colours and faces, in order."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MESH = ("vertices", "colors", "faces")
COUNTS = ("num_cubes", "num_faces_raw", "num_vertices_welded", "num_faces_clean", "num_faces", "num_vertices")


def _engine_with(xyz, sdf0, sdf_refined, weight, rgb, voxel_size):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    n = len(xyz)
    e.upload_grid(xyz, sdf0, sdf_refined, np.full(n, 0.6), weight, rgb, voxel_size)
    return e


def _check(e, g, source, lc):
    """the engine's mesh of its grid against mesh_ref on the downloaded grid"""
    import mesh_ref
    m = e.extract_mesh(source, lc)
    r = mesh_ref.extract_grid(g, source, lc)
    for k in MESH:
        assert m[k].shape == r[k].shape and m[k].tobytes() == r[k].tobytes(), (source, lc, k)
    got = {k: int(getattr(m["info"], k)) for k in COUNTS}
    assert got == r["info"], (got, r["info"])
    return m


def _check_all(e, sources=("fused", "refined")):
    g = e.download_grid()
    return [_check(e, g, src, lc) for src in sources for lc in (False, True)]


def test_tiny_scene_bytes_equal(tiny_scene):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(tiny_scene)
    ms = _check_all(e)
    assert len(ms[0]["faces"]) > 1000
    print({k: int(getattr(ms[0]["info"], k)) for k in COUNTS})


def test_constructed_grids_bytes_equal():
    import test_mesh as tm
    cases = {
        "opposite_ends": tm.opposite_end_grid(),
        "floaters": tm.two_blobs(1, 2),
        "tie": tm.two_blobs(1, 1),
        "sphere_far": tm.grid(tm._sphere((70000.37, 70000.61, 70000.23), 4.3)),
        "missing_111": tm.grid(tm.cube(1), drop=(tm.gen_mc_tables.CORNERS[4],)),
        "zero_weight": tm.grid(tm.cube(1), weight={tm.gen_mc_tables.CORNERS[6]: 0.0}),
        "empty": tm.grid(tm.cube(0)),
    }
    for zero in (0.0, 5e-6, -0.0):
        v = tm.cube(1 | 4 | 8)
        v[tm.gen_mc_tables.CORNERS[1]] = zero
        cases[f"near_zero_{zero}"] = tm.grid(v)
    v = tm.cube(255 - 16)
    v[tm.gen_mc_tables.CORNERS[4]] = 0.0
    cases["unused_vertex"] = tm.grid(v)
    for name, (xyz, sdf, w, rgb) in cases.items():
        # sdf0 and the refined sdf differ (opposite signs): the source switch must pick the right one
        e = _engine_with(xyz, -sdf, sdf, w, rgb, 1.0)
        ms = _check_all(e)
        print(name, [len(m["faces"]) for m in ms], [len(m["vertices"]) for m in ms])
    xyz, sdf, w, rgb = cases["opposite_ends"]
    e = _engine_with(xyz, sdf, sdf, w, rgb, 1.0)
    assert len(e.extract_mesh("refined")["vertices"]) == 8


def _fused_fixture_engine():
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.engine import Engine
    g = np.load(os.path.join(HERE, "golden", "tiny_fusion.npz"))
    p = engine.default_fusion_params()
    p.voxel_size, p.depth_min, p.depth_max, p.integration_weight_sample = (float(x) for x in g["params"])
    cam = tuple(g["cam"])
    e = Engine(0)
    e.fusion_begin(p)
    e.fusion_integrate(cam, g["depth"], cam, g["bgr"], g["c2w"], g["w2c"])
    assert e.fusion_finish() > 0
    return e


def test_fused_grid_bytes_equal():
    e = _fused_fixture_engine()
    ms = _check_all(e)
    assert len(ms[0]["faces"]) > 100


def _gn_params(s):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    return p


def test_after_gn_and_recolor_bytes_equal(tiny_scene):
    from intrinsic3d_b200.engine import Engine
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    e = Engine(0)
    e.load_scene(s)
    for _ in range(2):
        e.gn_iteration(_gn_params(s))
    e.upload_color_frames(make_color_frames(s))
    e.recompute_colors()
    g = e.download_grid()
    assert not np.array_equal(g["sdf0"], g["sdf_refined"])
    ms = _check_all(e)
    assert ms[0]["vertices"].tobytes() != ms[2]["vertices"].tobytes()     # fused and refined surfaces differ


def test_after_prune_upsample_bytes_equal(tiny_scene):
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    e = Engine(0)
    e.load_scene(s)
    e.extract_mesh()
    vs = float(s["voxel_size"])
    e.clear_voxels_outside_thin_shell(2.0 * vs)
    assert e.L.i3d_download_mesh(e.h, None, None, None) != 0          # pruning changed the voxel set
    e.upsample_grid()
    e.clear_voxels_outside_thin_shell(vs)
    e.upsample_grid()
    _check_all(e)


def test_many_components_bytes_equal(tiny_scene):
    """A noisy refined sdf scatters the surface into a few hundred face-connected components (deep union-find trees after the
    upsample): the filtered mesh, and the unfiltered one, against the restatement."""
    s = tiny_scene
    vs = float(s["voxel_size"])
    noisy = s["sdf0"] + np.random.default_rng(4).normal(0.0, 1.5 * vs, len(s["sdf0"]))
    e = _engine_with(s["xyz"], s["sdf0"], noisy, s["weight"], s["rgb"], vs)
    for upsample in (False, True):
        if upsample:
            e.upsample_grid()
        m = _check_all(e, sources=("refined",))
        assert m[1]["info"].num_faces < m[1]["info"].num_faces_clean          # the filter removed floaters
        print(e.n, {k: int(getattr(m[1]["info"], k)) for k in COUNTS})


def test_golden_fixture_bytes_equal():
    g = np.load(os.path.join(HERE, "golden", "tiny_mesh.npz"))
    e = _engine_with(g["xyz"], g["sdf0"], g["sdf_refined"], g["weight"], g["rgb"], float(g["voxel_size"]))
    for src in ("fused", "refined"):
        for lc in (0, 1):
            m = e.extract_mesh(src, bool(lc))
            for k in MESH:
                assert m[k].tobytes() == g[f"{src}_{lc}_{k}"].tobytes(), (src, lc, k)


def _mesh_bytes(m):
    return b"".join(m[k].tobytes() for k in MESH)


def test_c3_run_to_run_bit_identical():
    """Full C3 (2 M voxels) and one upsample (16 M): two extractions, and two engines, give byte-identical meshes."""
    import torch
    from intrinsic3d_b200.engine import Engine
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c3", device="cuda" if torch.cuda.is_available() else "cpu")
    engines = [Engine(0), Engine(0)]
    for e in engines:
        e.load_scene(s)
    for level in range(2):
        for src in ("fused", "refined"):
            for lc in (False, True):
                a = engines[0].extract_mesh(src, lc)
                b = engines[0].extract_mesh(src, lc)
                c = engines[1].extract_mesh(src, lc)
                assert _mesh_bytes(a) == _mesh_bytes(b) == _mesh_bytes(c), (level, src, lc)
                assert len(a["faces"]) > 100000
                if lc:                                         # the scene's surface is one component: the filter keeps every face
                    assert a["info"].num_faces == a["info"].num_faces_clean
                print(level, src, lc, engines[0].n, {k: int(getattr(a["info"], k)) for k in COUNTS})
        if level == 0:
            for e in engines:
                e.upsample_grid()
    for e in engines:
        e.close()


def test_gn_iteration_unchanged_by_extraction(tiny_scene):
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    out = []
    for extract in (False, True):
        e = Engine(0)
        e.load_scene(s)
        e.gn_iteration(_gn_params(s))
        if extract:
            e.extract_mesh("refined", True)
            e.extract_mesh("fused", False)
        info = e.gn_iteration(_gn_params(s))
        out.append((bytes(info)[:type(info).time_add.offset], e.download_state()))
    assert out[0][0] == out[1][0]
    for k in out[0][1]:
        assert out[0][1][k].tobytes() == out[1][1][k].tobytes(), k


def test_refusals_leave_engine_usable(tiny_scene):
    from intrinsic3d_b200.ctypes_defs import I3DMeshInfo, I3DMeshParams
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    info = I3DMeshInfo()
    assert e.L.i3d_extract_mesh(e.h, C.byref(I3DMeshParams(1, 0)), C.byref(info)) != 0
    assert "no grid" in e.L.i3d_last_error(e.h).decode()
    e.load_scene(tiny_scene)
    assert e.L.i3d_download_mesh(e.h, None, None, None) != 0
    assert "no mesh" in e.L.i3d_last_error(e.h).decode()
    for bad in (-1, 2):
        assert e.L.i3d_extract_mesh(e.h, C.byref(I3DMeshParams(bad, 0)), C.byref(info)) != 0
        assert "sdf_source" in e.L.i3d_last_error(e.h).decode()
    with pytest.raises(ValueError):
        e.extract_mesh("sdf0")
    m = e.extract_mesh("refined")
    assert len(m["faces"]) > 0
    e.upsample_grid()                                      # a new voxel set drops the resident mesh
    assert e.L.i3d_download_mesh(e.h, None, None, None) != 0
    assert len(e.extract_mesh("refined")["faces"]) > 0
