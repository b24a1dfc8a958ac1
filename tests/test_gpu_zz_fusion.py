"""GPU parity of the RGB-D fusion (i3d_fusion_begin / integrate / finish) against the float CPU oracle of tests/native/fusion_oracle.cpp.
Exact-rounding float and integer work: the bar is BIT-EXACT voxel sets, canonical order and every sdf / weight / colour byte."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
VOL = ("xyz", "sdf", "weight", "rgb")


def _scene():
    from intrinsic3d_b200.scene import make_scene
    return make_scene(radius_vox=16.0, frames=5, width=160, height=120, voxel_size=0.004, seed=3)


def _params(s, window=2, ws=10.0, clip=None, cap=0):
    from fusion_ref import depth_range
    from intrinsic3d_b200 import engine
    p = engine.default_fusion_params()
    p.voxel_size = float(s["voxel_size"])
    p.depth_min, p.depth_max = depth_range(s)
    p.integration_weight_sample = ws
    p.discont_window_size = window
    if clip is not None:
        for k in range(6):
            p.clip_bounds[k] = clip[k]
    p.initial_capacity = cap
    return p


def _oracle(p):
    from fusion_ref import FusionOracle
    return FusionOracle(p.voxel_size, p.depth_min, p.depth_max, p.integration_weight_sample, list(p.clip_bounds), p.discont_window_size,
                        p.correct_sdf_iterations)


def _inputs(s, frames=None, color_x2=False):
    from fusion_ref import scene_inputs
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    if color_x2:
        # a colour camera at twice the depth resolution with its own intrinsics
        W, H = dcam[0], dcam[1]
        ccam = (2 * W, 2 * H, 2.1 * dcam[2], 1.9 * dcam[3], 2 * dcam[4] + 3.5, 2 * dcam[5] - 2.0)
        bgr = np.repeat(np.repeat(bgr, 2, axis=1), 2, axis=2)
        bgr = (bgr.astype(np.int32) + np.arange(2 * W, dtype=np.int32)[None, None, :, None] % 7).clip(0, 255).astype(np.uint8)
    if frames is not None:
        depth, bgr, c2w, w2c = depth[:frames], bgr[:frames], c2w[:frames], w2c[:frames]
    return dcam, depth, ccam, bgr, c2w, w2c


def _fuse_engine(p, inp, e=None):
    from intrinsic3d_b200.engine import Engine
    e = e or Engine(0)
    e.fusion_begin(p)
    e.fusion_integrate(*inp)
    return e


def _same(a, b):
    for k in VOL:
        assert a[k].shape == b[k].shape, (k, a[k].shape, b[k].shape)
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), (k, int((a[k] != b[k]).sum()))


CASES = {
    "1frame": dict(frames=1),
    "all": dict(),
    "window0_ws0": dict(window=0, ws=0.0),
    "window2_ws0": dict(ws=0.0),
    "window0_ws10": dict(window=0),
    "clip_half": dict(clip=True),
    "color_x2": dict(color_x2=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_fusion_volume_bit_exact(case):
    c = CASES[case]
    s = _scene()
    clip = (-1.0, 1.0, -1.0, 0.0, -1.0, 1.0) if c.get("clip") else None     # y <= 0: half of the sphere
    p = _params(s, window=c.get("window", 2), ws=c.get("ws", 10.0), clip=clip)
    inp = _inputs(s, frames=c.get("frames"), color_x2=c.get("color_x2", False))
    e = _fuse_engine(p, inp)
    o = _oracle(p)
    assert o.integrate(*inp) == 0
    ve, vo = e.fusion_volume(), o.volume()
    assert len(vo["xyz"]) > 1000 and (vo["weight"] > 0).sum() > 500
    _same(ve, vo)
    if clip is not None:
        assert (vo["xyz"][:, 1] <= 1).all()
    print(f"{case}: {len(vo['xyz'])} voxels, {(vo['weight'] > 0).sum()} integrated")


def test_fusion_finish_bit_exact_against_jacobi_oracle():
    s = _scene()
    p = _params(s)
    inp = _inputs(s)
    e = _fuse_engine(p, inp)
    m = e.fusion_finish()
    g = e.download_grid()
    o = _oracle(p)
    assert o.integrate(*inp) == 0
    og = o.clone()
    sj, sg = o.finish(1), og.finish(2)
    vj, vg = o.volume(), og.volume()
    assert m == len(vj["xyz"]) > 1000
    assert np.array_equal(g["xyz"], vj["xyz"])
    assert np.array_equal(g["sdf0"], vj["sdf"].astype(np.float64)) and np.array_equal(g["sdf_refined"], g["sdf0"])
    assert np.array_equal(g["weight"].view(np.uint32), vj["weight"].view(np.uint32)) and np.array_equal(g["rgb"], vj["rgb"])
    assert (g["albedo"] == 0.6).all() and (g["weight"] > 0).all()
    assert g["voxel_size"] == np.float32(p.voxel_size)
    assert e.phase_count("fusion_sweeps") == sj
    same_gs = all(np.array_equal(vj[k], vg[k]) for k in VOL)
    print(f"finish: {m} voxels; Jacobi {sj} sweeps, Gauss-Seidel {sg} sweeps; equal to Gauss-Seidel: {same_gs}")


def test_fusion_growth_gives_identical_result():
    s = _scene()
    inp = _inputs(s)
    e1 = _fuse_engine(_params(s), inp)
    e2 = _fuse_engine(_params(s, cap=1024), inp)
    assert e1.phase_count("fusion_growths") == 0 and e2.phase_count("fusion_growths") >= 3
    _same(e1.fusion_volume(), e2.fusion_volume())
    assert e1.fusion_finish() == e2.fusion_finish()
    g1, g2 = e1.download_grid(), e2.download_grid()
    for k in ("xyz", "sdf0", "weight", "rgb"):
        assert np.array_equal(g1[k], g2[k]), k
    print(f"growth: {e2.phase_count('fusion_growths')} growths from 1024 slots")


def test_fusion_run_to_run_bytes():
    s = _scene()
    inp = _inputs(s)
    a, b = _fuse_engine(_params(s), inp), _fuse_engine(_params(s), inp)
    _same(a.fusion_volume(), b.fusion_volume())
    a.fusion_finish(), b.fusion_finish()
    ga, gb = a.download_grid(), b.download_grid()
    for k in ("xyz", "sdf0", "sdf_refined", "albedo", "weight", "rgb"):
        assert ga[k].tobytes() == gb[k].tobytes(), k


def test_fused_grid_feeds_the_path():
    """fused grid -> lighting estimate -> one GN residual build, against the parity oracle loaded with the downloaded fused grid."""
    import oracle
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.ctypes_defs import default_params
    s = _scene()
    e = _fuse_engine(_params(s), _inputs(s))
    e.fusion_finish()
    g = e.download_grid()
    e.upload_frames(s["lum"], s["depth"])
    e.set_camera(s["poses"], s["intr"], s["dist"])
    o = oracle.Oracle(threads=8)
    o.set_grid(g)
    o.set_frames(s["lum"], s["depth"])
    o.set_camera(s["poses"], s["intr"], s["dist"])
    shell = 2.0 * float(s["voxel_size"])
    le, lo = engine.default_lighting_params(), oracle.default_lighting_params()
    for lp in (le, lo):
        lp.thres_shell = shell; lp.subvolume_size = 0.04
    ie, io = e.estimate_lighting(le), o.estimate_lighting(lo)
    assert (ie.num_subvolumes, ie.num_data_rows, ie.lm_iterations) == (io.num_subvolumes, io.num_data_rows, io.lm_iterations)
    assert np.abs(e.download_lighting()[1] - o.lighting()[1]).max() <= 1e-8 * np.abs(o.lighting()[1]).max()
    p = default_params()
    p.thres_shell = shell
    p.build_only = 1
    je, jo = e.gn_iteration(p), o.gn_iteration(p)
    assert list(je.type_residuals) == list(jo.type_residuals) and jo.type_residuals[0] > 1000
    np.testing.assert_allclose(je.cost_initial, jo.cost_initial, rtol=1e-9)
    fe, we, ae = e.debug_observations(5)
    fo, wo, ao = o.observations(5)
    assert np.array_equal(ae, ao) and np.array_equal(fe, fo) and np.array_equal(we.view(np.uint32), wo.view(np.uint32))


def test_fusion_errors_leave_engine_usable():
    from intrinsic3d_b200.engine import Engine
    s = _scene()
    inp = _inputs(s, frames=2)
    e = Engine(0)
    with pytest.raises(RuntimeError, match="no fusion in progress"):
        e.fusion_integrate(*inp)
    p = _params(s)
    p.voxel_size = 1e-5
    with pytest.raises(RuntimeError, match="voxel_size"):
        e.fusion_begin(p)
    far = list(inp)
    c2w = inp[4].copy()
    c2w[:, 9] += 1.0e4                      # 10 km away: beyond the +-2^20 voxel range at 4 mm
    far[4] = c2w
    e.fusion_begin(_params(s))
    with pytest.raises(RuntimeError, match="coordinate range"):
        e.fusion_integrate(*far)
    with pytest.raises(RuntimeError, match="no fusion in progress"):
        e.fusion_finish()
    # a following fusion works and matches the oracle
    p = _params(s)
    _fuse_engine(p, inp, e)
    o = _oracle(p)
    assert o.integrate(*inp) == 0
    _same(e.fusion_volume(), o.volume())


def test_engine_matches_golden_fusion():
    import os
    from intrinsic3d_b200 import engine
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_fusion.npz"))
    p = engine.default_fusion_params()
    p.voxel_size, p.depth_min, p.depth_max, p.integration_weight_sample = (float(x) for x in g["params"])
    cam = tuple(g["cam"])
    e = _fuse_engine(p, (cam, g["depth"], cam, g["bgr"], g["c2w"], g["w2c"]))
    assert e.fusion_finish() == len(g["xyz"])
    d = e.download_grid()
    assert np.array_equal(d["xyz"], g["xyz"]) and np.array_equal(d["sdf0"], g["sdf"].astype(np.float64))
    assert np.array_equal(d["weight"], g["weight"]) and np.array_equal(d["rgb"], g["rgb"])
    assert e.phase_count("fusion_sweeps") == int(g["sweeps"])
