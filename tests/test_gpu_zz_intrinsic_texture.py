"""GPU tests of the texture decomposition and the relit raster (i3d_decompose_texture, i3d_download_intrinsic_texture,
i3d_set_relight, I3D_RASTER_COLOR_RELIT) against tests/intrinsic_texture_ref.py, each engine against the restatement of its own
downloaded subvolume SH.  Explicitly rounded float arithmetic and integer atomics: the bar is BYTE-EQUAL atlases, planes and counts."""
import numpy as np
import pytest

import intrinsic_texture_ref as it

pytestmark = pytest.mark.gpu
PLANES = ("depth", "face", "bary", "normal", "rgb")
SH = np.array([0.7, 0.12, -0.2, 0.15, 0.03, -0.05, 0.06, 0.02, -0.04], np.float32)


def _engine(s, subvolume_size=0.02):
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import make_color_frames
    e = engine.Engine(0)
    e.load_scene(s)
    col = make_color_frames(s)
    e.upload_color_frames(col)
    lp = engine.default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    lp.subvolume_size = subvolume_size
    e.estimate_lighting(lp)
    return e, col


def _cam(e):
    import render_ref as rr
    st = e.download_state()
    return rr.pose_rt(st["poses"]), rr.camera(st["intr"], st["dist"])


def _lighting(e, sh, subvolume_size):
    if sh is not None:
        return it.global_sh(sh)
    idx, sub = e.download_lighting()
    return it.estimate_sh(idx, sub, subvolume_size)


def _check(e, s, mesh, b, S, sh, subvolume_size, obs):
    g = e.decompose_texture(0.05, sh)
    r = it.decompose(b["image"], mesh, S, _lighting(e, sh, subvolume_size), 0.05, obs)
    assert g["albedo"].tobytes() == r["albedo"].tobytes() and g["shading"].tobytes() == r["shading"].tobytes()
    i = g["info"].as_dict()
    for k in it.INFO_COUNTS:
        assert i[k] == r["info"][k], (k, i[k], r["info"][k])
    assert [float(np.float32(x)) for x in i["albedo_min"]] == r["info"]["albedo_min"] and i["ms_decompose"] > 0
    assert [float(np.float32(x)) for x in i["albedo_max"]] == r["info"]["albedo_max"]
    assert i["num_texels_lit"] > 0
    return g


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_decomposition_byte_equal(name):
    from intrinsic3d_b200.scene import config_scene
    s = config_scene(name)
    for size in (0.02, 0.05):
        e, col = _engine(s, size)
        rt, cam = _cam(e)
        vs = float(s["voxel_size"])
        for cell in (None, 4):
            m = e.extract_mesh("refined", True)
            if cell:
                m = e.simplify_mesh(cell * vs)
            S = 8
            b = e.bake_texture(S)
            obs = it.observed(m, s["depth"], rt, cam, S)
            assert b["info"].num_texels_observed == int(obs.sum())
            for sh in (None, SH):
                _check(e, s, m, b, S, sh, size, obs)


def test_decomposition_byte_equal_c2():
    """C2, full and simplified at 4 voxels, estimate and global lighting.  The fallback count is checked against the bake's count (the
    restatement of the observation flags over 50 frames would dominate the run); every other count and both atlases byte-equal."""
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c2")
    e, col = _engine(s, 0.05)
    for cell in (None, 4):
        m = e.extract_mesh("refined", True)
        if cell:
            m = e.simplify_mesh(cell * float(s["voxel_size"]))
        b = e.bake_texture(6)
        for sh in (None, SH):
            g = e.decompose_texture(0.05, sh)
            r = it.decompose(b["image"], m, 6, _lighting(e, sh, 0.05), 0.05)
            assert g["albedo"].tobytes() == r["albedo"].tobytes() and g["shading"].tobytes() == r["shading"].tobytes()
            i = g["info"].as_dict()
            for k in it.INFO_COUNTS[:-1]:
                assert i[k] == r["info"][k], (k, i[k], r["info"][k])
            assert i["num_texels_lit_fallback"] <= b["info"].num_texels_fallback
            assert [float(np.float32(x)) for x in i["albedo_max"]] == r["info"]["albedo_max"]


def test_golden_fixture_on_the_device(tiny_scene):
    import hashlib
    import os
    from intrinsic3d_b200 import engine
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_intrinsic_texture.npz"))
    s = tiny_scene
    e, col = _engine(s, float(g["subvolume_size"]))
    m = e.extract_mesh("refined", True)
    assert m["faces"].tobytes() == g["faces"].tobytes()
    b = e.bake_texture(6)
    assert b["image"].tobytes() == g["image"].tobytes()
    d = e.decompose_texture(float(g["min_shading"]), g["sh"])
    assert d["albedo"].tobytes() == g["global_albedo"].tobytes() and d["shading"].tobytes() == g["global_shading"].tobytes()
    assert [d["info"].as_dict()[k] for k in it.INFO_COUNTS] == g["global_info"].tolist()
    assert np.array([list(d["info"].albedo_min), list(d["info"].albedo_max)], np.float32).tobytes() == g["global_range"].tobytes()
    e.set_relight(g["sh"])
    r = e.rasterize_keyframes(g["relit_ids"], "relit")
    assert r["rgb"].tobytes() == g["relit_rgb"].tobytes() and r["face"].tobytes() == g["relit_face"].tobytes()
    assert [[st["num_covered"], st["color_count"], *st["color_abs"], *st["color_sq"]] for st in r["stats"]] == g["relit_counts"].tolist()
    idx, sub = e.download_lighting()
    # the estimate case: byte-equal where the engine's lighting estimate equals the oracle's stored one (otherwise the engine is checked
    # against the restatement of its own SH by the tests above)
    if idx.tobytes() == g["sub_index"].astype(idx.dtype).tobytes() and sub.tobytes() == g["sub_sh"].tobytes():
        de = e.decompose_texture(float(g["min_shading"]))
        assert hashlib.sha256(de["albedo"].tobytes() + de["shading"].tobytes()).digest() == g["estimate_digest"].tobytes()
    del engine


def test_relit_raster_byte_equal_keyframes_views_binning_and_batch(tiny_scene):
    s = tiny_scene
    e, col = _engine(s)
    rt, cam = _cam(e)
    m = e.extract_mesh("refined", True)
    S = 8
    b = e.bake_texture(S)
    d = e.decompose_texture()
    ids = list(range(e.F))
    _, H, W = s["depth"].shape
    for sh in (None, SH, np.array([1, 0, 0, 0, 0, 0, 0, 0, 0], np.float32)):
        e.set_relight(sh)
        g = e.rasterize_keyframes(ids, "relit")
        r = it.rasterize(m, rt, cam, W, H, d["albedo"], S, _lighting(e, sh, 0.02), depth=s["depth"], bgr=col, ids=ids)
        for k in PLANES:
            assert g[k].tobytes() == r[k].tobytes(), k
        for a, c in zip(g["stats"], r["stats"]):
            for k in ("num_covered", "num_observed", "depth_count", "color_count", "color_abs", "color_sq"):
                assert a[k] == c[k], (k, a[k], c[k])
        e.set_raster_binning(False)
        e.set_raster_batch(1)
        off = e.rasterize_keyframes(ids, "relit")
        assert all(off[k].tobytes() == g[k].tobytes() for k in PLANES) and off["stats"] == g["stats"]
        e.set_raster_binning(True)
        e.set_raster_batch(0)
    # odd-sized new views
    e.set_relight(SH)
    poses = np.stack([rt[0], rt[3]]).astype(np.float32)
    for Wv, Hv in ((37, 29), (123, 77)):
        cv = dict(fx=0.9 * Wv, fy=0.9 * Wv, cx=(Wv - 1) / 2 + 0.3, cy=(Hv - 1) / 2 - 0.2, width=Wv, height=Hv)
        rc = dict(fx=np.float32(cv["fx"]), fy=np.float32(cv["fy"]), cx=np.float32(cv["cx"]), cy=np.float32(cv["cy"]), d=np.zeros(5, np.float32))
        g = e.rasterize_views(cv, poses, "relit")
        r = it.rasterize(m, poses, rc, Wv, Hv, d["albedo"], S, it.global_sh(SH))
        for k in PLANES:
            assert g[k].tobytes() == r[k].tobytes(), (Wv, k)


def test_determinism_c3():
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c3")
    outs, shs = [], []
    for _ in range(2):
        e, _ = _engine(s)
        e.extract_mesh("refined", True)
        e.bake_texture(8)
        a = e.decompose_texture()
        b = e.decompose_texture()
        assert a["albedo"].tobytes() == b["albedo"].tobytes() and a["shading"].tobytes() == b["shading"].tobytes()
        e.set_relight(None)
        ids = list(range(0, e.F, max(1, e.F // 8)))
        k1, k2 = e.rasterize_keyframes(ids, "relit"), e.rasterize_keyframes(ids, "relit")
        assert k1["rgb"].tobytes() == k2["rgb"].tobytes() and k1["stats"] == k2["stats"]
        outs.append((a, k1))
        shs.append(e.download_lighting()[1].tobytes())
        del e
    if shs[0] == shs[1]:
        assert outs[0][0]["albedo"].tobytes() == outs[1][0]["albedo"].tobytes()
        assert outs[0][1]["rgb"].tobytes() == outs[1][1]["rgb"].tobytes()


def _texture_bytes(e):
    """the texture (atlas, uv) and the decomposition (albedo, shading) on the device, as bytes"""
    import ctypes as C
    H, W = e._texture_hw
    F = e._texture_f
    rgb, uv = np.empty((H, W, 3), np.uint8), np.empty((F, 3, 2), np.float32)
    alb, sha = np.empty((H, W, 3), np.float32), np.empty((H, W), np.float32)
    e._check(e.L.i3d_download_texture(e.h, rgb.ctypes.data_as(C.POINTER(C.c_uint8)), uv.ctypes.data_as(C.POINTER(C.c_float))))
    e._check(e.L.i3d_download_intrinsic_texture(e.h, alb.ctypes.data_as(C.POINTER(C.c_float)), sha.ctypes.data_as(C.POINTER(C.c_float))))
    return rgb.tobytes() + uv.tobytes() + alb.tobytes() + sha.tobytes()


def test_refusals_and_lifetime(tiny_scene):
    from intrinsic3d_b200.engine import Engine
    s = tiny_scene
    e = Engine(0)
    e.load_scene(s)
    from intrinsic3d_b200.scene import make_color_frames
    e.upload_color_frames(make_color_frames(s))
    e.extract_mesh("refined", True)
    with pytest.raises(RuntimeError, match="no texture"):
        e.decompose_texture(sh=SH)
    tb = e.bake_texture(8)
    e._texture_hw, e._texture_f = tb["image"].shape[:2], len(tb["uv"])
    with pytest.raises(RuntimeError, match="lighting estimate"):
        e.decompose_texture()                                         # estimate source without an estimate
    with pytest.raises(RuntimeError, match="relit colour source needs a decomposition"):
        e.rasterize_keyframes([0], "relit")
    with pytest.raises(RuntimeError, match="min_shading"):
        e.decompose_texture(float("nan"), SH)
    with pytest.raises(RuntimeError, match="min_shading"):
        e.decompose_texture(-0.1, SH)
    bad = SH.copy()
    bad[4] = np.inf
    with pytest.raises(RuntimeError, match="not finite"):
        e.decompose_texture(0.05, bad)
    with pytest.raises(RuntimeError, match="not finite"):
        e.set_relight(bad)
    assert e.L.i3d_download_intrinsic_texture(e.h, None, None) != 0
    first = e.decompose_texture(0.05, SH)
    e.rasterize_keyframes([0, 1], "texture")
    planes = e._download_raster(2, *e.frame_size, 31)
    tex0 = _texture_bytes(e)
    # refusals leave the decomposition and the raster planes as they were
    for call in (lambda: e.decompose_texture(-1.0, SH), lambda: e.decompose_texture(0.05, bad), lambda: e.decompose_texture(0.05, None),
                 lambda: e.rasterize_keyframes([0], "relit")):
        with pytest.raises(RuntimeError):
            call()
    again = e._download_raster(2, *e.frame_size, 31)
    assert all(planes[k].tobytes() == again[k].tobytes() for k in planes)
    assert _texture_bytes(e) == tex0
    import ctypes as C
    alb = np.empty_like(first["albedo"])
    e._check(e.L.i3d_download_intrinsic_texture(e.h, alb.ctypes.data_as(C.POINTER(C.c_float)), None))
    assert alb.tobytes() == first["albedo"].tobytes()
    # a bad source is refused
    from intrinsic3d_b200.ctypes_defs import I3DIntrinsicTextureParams, I3DIntrinsicTextureInfo, I3DShLighting
    prm = I3DIntrinsicTextureParams(I3DShLighting(7, 0, (C.c_float * 9)()), 0.05, 0)
    assert e.L.i3d_decompose_texture(e.h, C.byref(prm), C.byref(I3DIntrinsicTextureInfo())) != 0
    assert e.L.i3d_set_relight(e.h, C.byref(I3DShLighting(7, 0, (C.c_float * 9)()))) != 0
    # a new bake drops the decomposition; so do a simplification and an extraction
    e.set_relight(SH)
    e.rasterize_keyframes([0], "relit")
    e.bake_texture(8)
    with pytest.raises(RuntimeError, match="decomposition"):
        e.rasterize_keyframes([0], "relit")
    e.decompose_texture(0.05, SH)
    e.simplify_mesh(4 * float(s["voxel_size"]))
    with pytest.raises(RuntimeError, match="no texture"):
        e.decompose_texture(0.05, SH)
    with pytest.raises(RuntimeError, match="decomposition"):
        e.rasterize_keyframes([0], "relit")
    # a later lighting estimate does not update the decomposition
    from intrinsic3d_b200 import engine
    e.extract_mesh("refined", True)
    e.bake_texture(8)
    d0 = e.decompose_texture(0.05, SH)
    lp = engine.default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    e.estimate_lighting(lp)
    alb = np.empty_like(d0["albedo"])
    e._check(e.L.i3d_download_intrinsic_texture(e.h, alb.ctypes.data_as(C.POINTER(C.c_float)), None))
    assert alb.tobytes() == d0["albedo"].tobytes()
    e.set_relight(None)
    e.rasterize_keyframes([0], "relit")                                # the estimate exists now


def test_unchanged_state(tiny_scene):
    """A GN iteration, a recolouring, a bake, a texture raster and the next extraction are byte-identical with and without the new calls."""
    from intrinsic3d_b200 import engine
    s = tiny_scene
    res = []
    for extra in (False, True):
        e, col = _engine(s)
        e.extract_mesh("refined", True)
        e.bake_texture(8)
        if extra:
            e.decompose_texture()
            e.set_relight(SH)
            e.rasterize_keyframes([0, 1], "relit")
        p = engine.default_params()
        p.thres_shell = s["thres_shell"]
        p.forced_cg_iterations = 4
        e.gn_iteration(p)
        e.recompute_colors()
        m = e.extract_mesh("refined", True)
        b = e.bake_texture(8)
        r = e.rasterize_keyframes([0, 1, 2], "texture")
        st = e.download_state()
        res.append((m["vertices"].tobytes(), m["colors"].tobytes(), b["image"].tobytes(), r["rgb"].tobytes(),
                    *(np.asarray(v).tobytes() for v in st.values())))
    assert res[0] == res[1]
