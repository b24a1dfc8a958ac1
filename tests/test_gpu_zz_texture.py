"""GPU tests of the texture bake (i3d_bake_texture, i3d_download_texture) against the numpy restatement tests/texture_ref.py.  Explicitly
rounded float arithmetic and integer atomics only: the bar is BYTE-EQUAL atlases and UVs, and equal counts."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _engine(s, col):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(s)
    e.upload_color_frames(col)
    return e


def _ref_camera(e):
    import render_ref as rr
    st = e.download_state()
    return rr.pose_rt(st["poses"]), rr.camera(st["intr"], st["dist"])


def _check(e, s, col, mesh, S=12, occlusion=0.02, K=5, pose_rt=None):
    """bakes the resident mesh (`mesh` as downloaded) on the engine and with the restatement; byte-equal, equal counts"""
    import texture_ref as tr
    rt, cam = _ref_camera(e)
    if pose_rt is not None:
        rt = pose_rt
    r = tr.bake(mesh, s["depth"], col, rt, cam, S, occlusion, K)
    g = e.bake_texture(S, occlusion, K, pose_rt=pose_rt)
    assert g["image"].tobytes() == r["image"].tobytes(), (S, K, occlusion)
    assert g["uv"].tobytes() == r["uv"].tobytes()
    got = {k: int(getattr(g["info"], k)) for k in tr.INFO_COUNTS}
    assert got == r["info"], (got, r["info"])
    i = g["info"]
    assert 0 < i.num_texel_frames_visited <= i.num_texel_frames_total and i.ms_bake > 0
    return g


def _colour_scene(name="tiny", distort=False):
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = dict(config_scene(name))
    if distort:
        s["dist"] = np.array([0.03, -0.01, 0.004, 0.002, -0.0015])
    return s, make_color_frames(s)


def _gn_params(s):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    return p


def test_tiny_sources_modes_k_and_poses(tiny_scene):
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    e = _engine(s, col)
    e.gn_iteration(_gn_params(s))                       # a refined camera and sdf that differ from the fused ones
    e.recompute_colors(0.02, 5)
    vs = float(s["voxel_size"])
    for src in ("fused", "refined"):
        m = e.extract_mesh(src, True)
        for K in (0, 1, 5, 8):
            _check(e, s, col, m, 12, 0.02, K)
    _check(e, s, col, m, 7, 0.0, 5)                     # the occlusion test off
    m = e.extract_mesh("refined", False, "normals")     # a colour-mode mesh: its vertex colours feed the fallback
    _check(e, s, col, m, 6, 0.02, 5)
    m = e.simplify_mesh(4 * vs)
    _check(e, s, col, m, 12, 0.02, 5)
    import render_ref as rr
    rt = rr.pose_rt(s["poses_true"])                    # explicit poses
    _check(e, s, col, m, 9, 0.02, 3, pose_rt=rt)


def test_distortion_and_small_scene(small_scene):
    s, col = _colour_scene("tiny", distort=True)
    e = _engine(s, col)
    _check(e, s, col, e.extract_mesh("refined", True), 12, 0.02, 5)
    from intrinsic3d_b200.scene import make_color_frames
    s = small_scene
    col = make_color_frames(s)
    e = _engine(s, col)
    m = e.extract_mesh("refined", False)
    _check(e, s, col, m, 8, 0.02, 5)
    _check(e, s, col, e.simplify_mesh(2 * float(s["voxel_size"])), 12, 0.02, 0)


def test_c2_simplified():
    import torch
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = config_scene("c2", device="cuda" if torch.cuda.is_available() else "cpu")
    col = make_color_frames(s)
    e = _engine(s, col)
    e.extract_mesh("refined", True)
    m = e.simplify_mesh(4 * float(s["voxel_size"]))
    g = _check(e, s, col, m, 8, 0.02, 5)
    print("c2", len(m["faces"]), {k: getattr(g["info"], k) for k in ("num_texels_observed", "num_texels_fallback", "num_texel_frames_visited",
                                                                      "num_texel_frames_total", "ms_bake")})


_NO_CULL_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import numpy as np
from intrinsic3d_b200.scene import config_scene, make_color_frames
from intrinsic3d_b200.engine import Engine
s = config_scene("small"); col = make_color_frames(s)
e = Engine(0); e.load_scene(s); e.upload_color_frames(col)
e.extract_mesh("refined", False)
out = {{}}
for K in (0, 5):
    g = e.bake_texture(12, 0.02, K)
    out[f"{{K}}_image"], out[f"{{K}}_uv"] = g["image"], g["uv"]
    out[f"{{K}}_visited"] = np.int64(g["info"].num_texel_frames_visited)
np.savez(sys.argv[1], **out)
"""


def test_byte_equal_without_culling(tmp_path):
    """I3D_NO_CULL is read once per process: both runs in subprocesses"""
    res = []
    for env_extra in ({}, {"I3D_NO_CULL": "1"}):
        path = tmp_path / f"r{len(res)}.npz"
        env = dict(os.environ)
        env.pop("I3D_NO_CULL", None)
        env.update(env_extra)
        subprocess.check_call([sys.executable, "-c", _NO_CULL_SCRIPT.format(root=ROOT, tests=HERE), str(path)], env=env)
        res.append(np.load(path))
    for K in (0, 5):
        assert res[0][f"{K}_image"].tobytes() == res[1][f"{K}_image"].tobytes()
        assert res[0][f"{K}_uv"].tobytes() == res[1][f"{K}_uv"].tobytes()
    assert int(res[0]["5_visited"]) < int(res[1]["5_visited"])                 # the culling did skip frames


def test_c3_run_to_run_bit_identical():
    import torch
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = config_scene("c3", device="cuda" if torch.cuda.is_available() else "cpu")
    col = make_color_frames(s)
    engines = [_engine(s, col), _engine(s, col)]
    for cell in (None, 4):
        res = []
        for e in (engines[0], engines[0], engines[1]):
            e.extract_mesh("refined", False)
            if cell:
                e.simplify_mesh(cell * float(s["voxel_size"]))
            res.append(e.bake_texture(8 if cell is None else 12))
        assert res[0]["image"].tobytes() == res[1]["image"].tobytes() == res[2]["image"].tobytes(), cell
        assert res[0]["uv"].tobytes() == res[1]["uv"].tobytes() == res[2]["uv"].tobytes(), cell
        assert bytes(res[0]["info"])[:-8] == bytes(res[1]["info"])[:-8] == bytes(res[2]["info"])[:-8]      # all but ms_bake
        print("c3", cell, {k: getattr(res[0]["info"], k) for k in ("atlas_width", "num_faces", "num_texels_observed", "ms_bake")})
    for e in engines:
        e.close()


def test_golden_fixture(tiny_scene):
    from intrinsic3d_b200.scene import make_color_frames
    g = np.load(os.path.join(HERE, "golden", "tiny_texture.npz"))
    e = _engine(tiny_scene, make_color_frames(tiny_scene))
    m = e.extract_mesh("refined", True)
    assert m["faces"].tobytes() == g["faces"].tobytes()
    for k, (S, K) in enumerate(g["cases"]):
        t = e.bake_texture(int(S), float(g["occlusion"]), int(K))
        assert t["image"].tobytes() == g[f"{k}_image"].tobytes() and t["uv"].tobytes() == g[f"{k}_uv"].tobytes(), k


def _resident(e):
    from intrinsic3d_b200.engine import _p
    V, F = 100000, 200000
    out = dict(v=np.zeros((V, 3), np.float32), c=np.zeros((V, 3), np.uint8), f=np.zeros((F, 3), np.int32))
    assert e.L.i3d_download_mesh(e.h, _p(out["v"], C.c_float), _p(out["c"], C.c_uint8), _p(out["f"], C.c_int32)) == 0
    return b"".join(a.tobytes() for a in out.values())


def test_refusals_leave_mesh_and_texture(tiny_scene, small_scene):
    from intrinsic3d_b200.ctypes_defs import I3DTextureInfo, I3DTextureParams
    from intrinsic3d_b200.engine import Engine, default_texture_params
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    info = I3DTextureInfo()

    def bake(e, S=12, occ=0.02, K=5):
        return e.L.i3d_bake_texture(e.h, C.byref(I3DTextureParams(S, occ, K, 0)), None, C.byref(info))

    def err(e):
        return e.L.i3d_last_error(e.h).decode()
    e = Engine(0)
    e.load_scene(s)
    assert bake(e) != 0 and "no mesh" in err(e)
    e.extract_mesh("refined", True)
    assert bake(e) != 0 and "colour frames" in err(e)                           # no colour frames yet
    e.upload_color_frames(col)
    assert e.L.i3d_bake_texture(e.h, None, None, C.byref(info)) != 0
    assert e.L.i3d_download_texture(e.h, None, None) != 0 and "no texture" in err(e)
    first = e.bake_texture()
    mesh0 = _resident(e)
    for args, msg in (((5,), "texels_per_face"), ((257,), "texels_per_face"), ((12, 0.02, -1), "max_num_observations"),
                      ((12, 0.02, 9), "max_num_observations"), ((12, float("nan")), "finite"), ((12, float("inf")), "finite")):
        assert bake(e, *args) != 0, args
        assert msg in err(e), (args, err(e))
        assert _resident(e) == mesh0
        img = np.zeros_like(first["image"])
        assert e.L.i3d_download_texture(e.h, img.ctypes.data_as(C.POINTER(C.c_uint8)), None) == 0         # the previous texture stays
        assert img.tobytes() == first["image"].tobytes()
    assert e.bake_texture()["image"].tobytes() == first["image"].tobytes()
    with pytest.raises(RuntimeError):
        e.bake_texture(texels_per_face=3)
    # an atlas side above I3D_TEXTURE_MAX_SIDE: 15 k faces at 256 texels per face need 88 cells of 256 texels per row
    e2 = _engine(small_scene, make_color_frames(small_scene))
    e2.extract_mesh("refined", False)
    mesh2 = _resident(e2)
    assert bake(e2, 256) != 0 and "I3D_TEXTURE_MAX_SIDE" in err(e2) and _resident(e2) == mesh2
    assert e2.L.i3d_download_texture(e2.h, None, None) != 0
    # a mesh without faces: a sphere in the positive octant simplified with one cell
    import test_gpu_zz_mesh as tgm
    import test_mesh as tm
    xyz, sdf, w, rgb = tm.grid(tm._sphere((3.3, 2.6, 4.1), 2.2, half=4))
    e3 = tgm._engine_with(xyz, sdf, sdf, w, rgb, 0.004)
    e3.extract_mesh("refined")
    assert len(e3.simplify_mesh(1.0)["faces"]) == 0
    assert bake(e3) != 0 and "no faces" in err(e3)
    # struct sizes and defaults
    p = default_texture_params()
    assert (p.texels_per_face, p.max_num_observations, p.reserved) == (12, 5, 0) and abs(p.max_occlusion_distance - 0.02) < 1e-9
    assert e.L.i3d_sizeof_texture_params() == C.sizeof(I3DTextureParams) == 16
    assert e.L.i3d_sizeof_texture_info() == C.sizeof(I3DTextureInfo) == 80


def test_texture_dropped_by_extract_simplify_upsample(tiny_scene):
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    e = _engine(s, make_color_frames(s))
    for step in ("extract", "simplify", "upsample"):
        e.extract_mesh("refined", True)
        e.bake_texture(8)
        assert e.L.i3d_download_texture(e.h, None, None) == 0
        if step == "extract":
            e.extract_mesh("refined", True)
        elif step == "simplify":
            e.simplify_mesh(3 * float(s["voxel_size"]))
        else:
            e.upsample_grid()
        assert e.L.i3d_download_texture(e.h, None, None) != 0, step


def test_state_unchanged_by_bake(tiny_scene):
    """A GN iteration, a recolouring, a render and the next extraction are byte-identical with and without a bake in between."""
    from intrinsic3d_b200.scene import make_color_frames
    s = tiny_scene
    col = make_color_frames(s)
    out = []
    for bake in (False, True):
        e = _engine(s, col)
        e.gn_iteration(_gn_params(s))
        e.extract_mesh("refined", True)
        if bake:
            e.bake_texture(12, 0.02, 5)
            e.bake_texture(6, 0.0, 8)
        info = e.gn_iteration(_gn_params(s))
        cnt = e.recompute_colors(0.02, 5)
        r = e.render_keyframes([0, 1])
        m = e.extract_mesh("fused", False)
        out.append((bytes(info)[:type(info).time_add.offset], e.download_state(), cnt, e.download_colors(), r, m))
    assert out[0][0] == out[1][0] and out[0][2] == out[1][2]
    for k in out[0][1]:
        assert out[0][1][k].tobytes() == out[1][1][k].tobytes(), k
    assert out[0][3].tobytes() == out[1][3].tobytes()
    for k in out[0][4]:
        if k != "stats":
            assert out[0][4][k].tobytes() == out[1][4][k].tobytes(), k
    for k in ("vertices", "colors", "faces"):
        assert out[0][5][k].tobytes() == out[1][5][k].tobytes(), k
