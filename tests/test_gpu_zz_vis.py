"""GPU tests of the mesh colour modes (i3d_mode_colors / i3d_extract_mesh_colored) against the numpy restatement tests/vis_ref.py and,
for the meshes, tests/mesh_ref.py on the grid with the restated colours.  Exact-rounding float work and truncating casts: the bar is
BYTE-EQUAL colours, vertices and faces."""
import ctypes as C
import os

import numpy as np
import pytest

import vis_ref

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MESH = ("vertices", "colors", "faces")
SHADING = ("shading_sv", "shading_sv_const")


def _gn_params(s):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    return p


def _light(e, thres_shell, subvolume_size):
    from intrinsic3d_b200 import engine
    lp = engine.default_lighting_params()
    lp.thres_shell = thres_shell
    lp.subvolume_size = subvolume_size
    e.estimate_lighting(lp)


def _lit_engine(s, subvolume_size=0.02, gn=2):
    """the tiny scene after a lighting estimate and `gn` GN iterations: the refined sdf differs from sdf0 and the albedo varies"""
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(s)
    _light(e, s["thres_shell"], subvolume_size)
    for _ in range(gn):
        e.gn_iteration(_gn_params(s))
    return e


def _ref(e, g, mode, source, subvolume_size):
    idx, sh = e.download_lighting()
    return vis_ref.colors(g, mode, source, idx, sh, subvolume_size)


def test_mode_colors_bytes_equal(tiny_scene):
    e = _lit_engine(tiny_scene)
    g = e.download_grid()
    assert not np.array_equal(g["sdf0"], g["sdf_refined"]) and len(np.unique(g["albedo"])) > 1
    assert e.L.i3d_lighting_num_subvolumes(e.h) > 1
    for src in ("fused", "refined"):
        for mode in vis_ref.MODES:
            got = e.mode_colors(mode, src)
            want = _ref(e, g, mode, src, 0.02)
            assert got.shape == want.shape and got.tobytes() == want.tobytes(), (src, mode, int((got != want).any(1).sum()))
            if mode:
                assert e.phase_ms("mesh_colorize") > 0.0
    # the modes are not trivial on this grid
    assert len({e.mode_colors(m).tobytes() for m in vis_ref.MODES}) == len(vis_ref.MODES)


def test_single_subvolume_bytes_equal(tiny_scene):
    """the tiny grid moved into the positive octant, lit with 100 m subvolumes: one subvolume, whose SH the shading modes take as it is"""
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    rng = np.random.default_rng(3)
    n = len(s["xyz"])
    e = Engine(0)
    e.upload_grid(s["xyz"] + 1000, s["sdf0"], s["sdf0"] + rng.normal(0.0, 0.2 * float(s["voxel_size"]), n), 0.6 + 0.2 * rng.random(n),
                  s["weight"], s["rgb"], s["voxel_size"])
    _light(e, s["thres_shell"], 100.0)
    assert e.L.i3d_lighting_num_subvolumes(e.h) == 1
    g = e.download_grid()
    for mode in SHADING:
        for src in ("fused", "refined"):
            assert e.mode_colors(mode, src).tobytes() == _ref(e, g, mode, src, 100.0).tobytes(), (mode, src)


def test_meshes_bytes_equal(tiny_scene):
    import mesh_ref
    from intrinsic3d_b200.ctypes_defs import I3DMeshInfo, I3DMeshParams
    e = _lit_engine(tiny_scene)
    g = e.download_grid()
    for src in ("fused", "refined"):
        sdf = g["sdf_refined"] if src == "refined" else g["sdf0"]
        for mode in vis_ref.MODES:
            cols = _ref(e, g, mode, src, 0.02)
            for lc in (False, True):
                m = e.extract_mesh(src, lc, mode)
                r = mesh_ref.extract(g["xyz"], sdf, g["weight"], cols, g["voxel_size"], lc)
                for k in MESH:
                    assert m[k].shape == r[k].shape and m[k].tobytes() == r[k].tobytes(), (src, mode, lc, k)
    # mode 0 through the new call is i3d_extract_mesh
    plain = e.extract_mesh("refined", True)
    info = I3DMeshInfo()
    assert e.L.i3d_extract_mesh_colored(e.h, C.byref(I3DMeshParams(1, 1)), 0, C.byref(info)) == 0
    V, F = int(info.num_vertices), int(info.num_faces)
    out = dict(vertices=np.empty((V, 3), np.float32), colors=np.empty((V, 3), np.uint8), faces=np.empty((F, 3), np.int32))
    assert e.L.i3d_download_mesh(e.h, out["vertices"].ctypes.data_as(C.POINTER(C.c_float)), out["colors"].ctypes.data_as(C.POINTER(C.c_uint8)),
                                 out["faces"].ctypes.data_as(C.POINTER(C.c_int32))) == 0
    for k in MESH:
        assert out[k].tobytes() == plain[k].tobytes(), k


def test_golden_fixture():
    from intrinsic3d_b200.engine import Engine
    from intrinsic3d_b200.scene import config_scene
    f = np.load(os.path.join(HERE, "golden", "tiny_vis.npz"))
    e = Engine(0)
    e.upload_grid(f["xyz"], f["sdf0"], f["sdf_refined"], f["albedo"], f["weight"], f["rgb"], float(f["voxel_size"]))
    for src in ("fused", "refined"):
        for mode in vis_ref.MODES:
            if mode not in SHADING:
                assert e.mode_colors(mode, src).tobytes() == f[f"{src}_{mode or 'voxel'}"].tobytes(), (src, mode)
    # the device's own lighting estimate: the same subvolumes as the oracle's, and the colours of its SH as the restatement gives them
    _light(e, config_scene("tiny")["thres_shell"], float(f["subvolume_size"]))
    idx, sh = e.download_lighting()
    assert idx.tobytes() == f["sub_index"].tobytes() and np.abs(sh - f["sub_sh"]).max() <= 1e-8 * np.abs(f["sub_sh"]).max()
    g = e.download_grid()
    for src in ("fused", "refined"):
        for mode in SHADING:
            assert e.mode_colors(mode, src).tobytes() == vis_ref.colors(g, mode, src, idx, sh, float(f["subvolume_size"])).tobytes(), (src, mode)


def test_state_untouched(tiny_scene):
    """coloured extractions change neither the voxel colours nor a following GN iteration"""
    s = tiny_scene
    out = []
    for colour in (False, True):
        e = _lit_engine(s, gn=0)
        # the scene's per-voxel SH for the iterations: the lighting estimate sums with double atomics, so its last bits may differ
        # between the two engines; the subvolume SH it leaves only feed the shading modes
        e.set_sh(s["sh"])
        e.gn_iteration(_gn_params(s))
        rgb0 = e.download_colors()
        if colour:
            for mode in vis_ref.MODES:
                e.extract_mesh("refined", True, mode)
                e.mode_colors(mode, "fused")
            assert e.download_colors().tobytes() == rgb0.tobytes()
        info = e.gn_iteration(_gn_params(s))
        out.append((bytes(info)[:type(info).time_add.offset], e.download_state(), e.download_colors()))
    assert out[0][0] == out[1][0]
    for k in out[0][1]:
        assert out[0][1][k].tobytes() == out[1][1][k].tobytes(), k
    assert out[0][2].tobytes() == out[1][2].tobytes()


def test_refusals_leave_engine_usable(tiny_scene):
    from intrinsic3d_b200.ctypes_defs import I3DMeshInfo, I3DMeshParams
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    info = I3DMeshInfo()
    buf = np.empty((len(tiny_scene["xyz"]), 3), np.uint8)
    pbuf = buf.ctypes.data_as(C.POINTER(C.c_uint8))

    def err():
        return e.L.i3d_last_error(e.h).decode()

    assert e.L.i3d_extract_mesh_colored(e.h, C.byref(I3DMeshParams(1, 0)), 5, C.byref(info)) != 0 and "no grid" in err()
    assert e.L.i3d_mode_colors(e.h, 1, 5, pbuf) != 0 and "no grid" in err()
    e.load_scene(tiny_scene)                                    # per-voxel SH from i3d_set_sh, no lighting estimate
    for bad in (-1, 9):
        assert e.L.i3d_extract_mesh_colored(e.h, C.byref(I3DMeshParams(1, 0)), bad, C.byref(info)) != 0 and "color_mode" in err()
        assert e.L.i3d_mode_colors(e.h, 1, bad, pbuf) != 0 and "color_mode" in err()
    for bad in (-1, 2):
        assert e.L.i3d_extract_mesh_colored(e.h, C.byref(I3DMeshParams(bad, 0)), 5, C.byref(info)) != 0 and "sdf_source" in err()
        assert e.L.i3d_mode_colors(e.h, bad, 5, pbuf) != 0 and "sdf_source" in err()
    assert e.L.i3d_mode_colors(e.h, 1, 5, None) != 0 and "NULL" in err()
    for mode in (6, 7):
        assert e.L.i3d_extract_mesh_colored(e.h, C.byref(I3DMeshParams(1, 0)), mode, C.byref(info)) != 0 and "lighting" in err()
        assert e.L.i3d_mode_colors(e.h, 0, mode, pbuf) != 0 and "lighting" in err()
    for mode in ("subvol", "subvol_interp", "bogus"):
        with pytest.raises(ValueError):
            e.extract_mesh("refined", False, mode)
        with pytest.raises(ValueError):
            e.mode_colors(mode)
    # still usable: every other mode works, and after a lighting estimate the shading modes too
    g = e.download_grid()
    for mode in ("albedo", "normals", "chroma"):
        assert len(e.extract_mesh("refined", False, mode)["faces"]) > 0
        assert e.mode_colors(mode).tobytes() == vis_ref.colors(g, mode).tobytes()
    _light(e, tiny_scene["thres_shell"], 0.02)
    assert len(e.extract_mesh("refined", True, "shading_sv")["faces"]) > 0
    # a prune changes the voxel set and drops the lighting: the shading modes are refused again
    e.clear_voxels_outside_thin_shell(2.0 * float(tiny_scene["voxel_size"]))
    with pytest.raises(RuntimeError, match="lighting"):
        e.extract_mesh("refined", False, "shading_sv")
    with pytest.raises(RuntimeError, match="lighting"):
        e.mode_colors("shading_sv_const")
    assert len(e.extract_mesh("refined", False, "albedo")["faces"]) > 0


def _mesh_bytes(m):
    return b"".join(m[k].tobytes() for k in MESH)


def test_c3_run_to_run_bit_identical():
    """Full C3 (2 M voxels): two coloured extractions, and two engines, give byte-identical meshes for albedo and shading_sv."""
    import torch
    from intrinsic3d_b200.engine import Engine
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c3", device="cuda" if torch.cuda.is_available() else "cpu")
    engines = [Engine(0), Engine(0)]
    for e in engines:
        e.load_scene(s)
        _light(e, s["thres_shell"], 0.2)
    # the two engines' lighting estimates (double atomics) may differ in the last bits; the shading meshes of the two engines are
    # compared when the subvolume SH agree byte for byte, and otherwise each engine's colours are checked against the restatement
    same_sh = engines[0].download_lighting()[1].tobytes() == engines[1].download_lighting()[1].tobytes()
    print("subvolume SH of the two engines byte-identical:", same_sh)
    for mode in ("albedo", "shading_sv"):
        cross = mode == "albedo" or same_sh
        for lc in (False, True):
            a = engines[0].extract_mesh("refined", lc, mode)
            b = engines[0].extract_mesh("refined", lc, mode)
            c = engines[1].extract_mesh("refined", lc, mode)
            assert _mesh_bytes(a) == _mesh_bytes(b), (mode, lc)
            assert _mesh_bytes(a) == _mesh_bytes(c) or not cross, (mode, lc)
            assert len(a["faces"]) > 100000
        if cross:
            assert engines[0].mode_colors(mode).tobytes() == engines[1].mode_colors(mode).tobytes()
        else:
            g = engines[1].download_grid()
            assert engines[1].mode_colors(mode).tobytes() == _ref(engines[1], g, mode, "refined", 0.2).tobytes()
    for e in engines:
        e.close()
