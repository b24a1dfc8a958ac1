"""CPU tests of tests/render_ref.py, the numpy float32 restatement of the keyframe renderer (DESIGN.md §6m): planes with known answers,
the synthetic scene's analytic truth, the inverse lens distortion, and the pinned fixture tests/golden/tiny_render.npz."""
import os

import numpy as np

import render_ref as rr

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32


def plane_grid(normal, offset, half=12, band=3.0, vs=0.01):
    """Every voxel of a (2 half + 1)^3 block within `band` voxels of the plane n . p = offset (metres), sdf = offset - n . p (positive on
    the side the camera at the origin looks from)."""
    n = np.asarray(normal, np.float64)
    n /= np.linalg.norm(n)
    r = np.arange(-half, half + 1)
    X, Y, Z = np.meshgrid(r, r, r + int(round(offset / vs)), indexing="ij")
    xyz = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1).astype(np.int32)
    sdf = offset - (xyz.astype(np.float64) * float(f32(vs))) @ n
    keep = np.abs(sdf) <= band * vs
    xyz, sdf = xyz[keep], sdf[keep]
    m = len(xyz)
    return dict(xyz=xyz, sdf0=sdf, sdf_refined=sdf, albedo=np.full(m, 0.5), weight=np.ones(m, f32), rgb=np.full((m, 3), 128, np.uint8),
                voxel_size=f32(vs))


def _identity_view(g, W=24, H=20, f=40.0, dist=np.zeros(5)):
    grid = rr.grid_of(g, "refined")
    cam = rr.camera([f, f, (W - 1) / 2.0, (H - 1) / 2.0], dist)
    rt = rr.pose_rt(np.zeros((1, 6)))[0]
    return rr.render_view(grid, rt, cam, W, H, photometric=False), cam, rt


def test_plane_head_on_exact():
    g = plane_grid((0, 0, 1), 0.3)
    v, _, _ = _identity_view(g)
    assert v["hit"].all()
    # measured: max |depth - 0.3| = 3.0e-8 m (one float ulp), normals exactly (0, 0, -1)
    assert np.abs(v["depth"] - f32(0.3)).max() <= 1e-7
    assert np.array_equal(v["normal"].reshape(-1, 3), np.tile(np.array([0, 0, -1], f32), (v["hit"].size, 1)))
    assert np.all(v["albedo"] == f32(0.5))


def test_plane_at_an_angle():
    nrm = np.array([0.3, -0.2, 1.0])
    nrm /= np.linalg.norm(nrm)
    g = plane_grid(nrm, 0.3)
    v, cam, rt = _identity_view(g)
    assert v["hit"].all()
    # the exact depth of the plane along each pixel's ray: z = offset / (n . (x, y, 1))
    u, w = np.meshgrid(np.arange(24), np.arange(20))
    x, y = (u - cam["cx"]) / cam["fx"], (w - cam["cy"]) / cam["fy"]
    z = 0.3 / (nrm[0] * x + nrm[1] * y + nrm[2])
    err = np.abs(v["depth"] - z).max()
    nerr = np.abs(v["normal"] + nrm[None, None, :]).max()
    # measured: depth 5.4e-8 m, normal 5.6e-8 (trilinear interpolation of a linear sdf is exact up to float rounding)
    assert err <= 2e-7 and nerr <= 2e-7, (err, nerr)


def test_non_finite_pose_has_no_samples():
    """A NaN or infinite pose gives a view without hits (and the march ends)."""
    g = plane_grid((0, 0, 1), 0.3)
    grid = rr.grid_of(g, "refined")
    cam = rr.camera([40.0, 40.0, 11.5, 9.5], np.zeros(5))
    for bad in ([np.nan, 0, 0, 0, 0, 0], [0, 0, 0, 0, np.inf, 0]):
        v = rr.render_view(grid, rr.pose_rt(np.array([bad], np.float64))[0], cam, 24, 20, photometric=False)
        assert not v["hit"].any() and not v["depth"].any()


def _truth_scene():
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("tiny", albedo_const=0.6)
    return s


def test_truth_against_the_analytic_renderer():
    """sdf_refined = sdf_true, constant albedo, the scene's global SH, rendered at poses_true: depth and luminance against the scene's
    analytic ray-marched images, on the pixels both hit."""
    s = _truth_scene()
    g = dict(xyz=s["xyz"], sdf0=s["sdf0"], sdf_refined=s["sdf_true"], albedo=s["albedo"], weight=s["weight"], voxel_size=s["voxel_size"])
    grid = rr.grid_of(g, "refined", s["sh"], np.ones(len(s["xyz"]), np.uint8))
    ids = [0, 3]
    out = rr.render(grid, s["poses_true"], s["intr"], s["dist"], 1.0, ids, s["depth"], s["lum"])
    vs = float(s["voxel_size"])
    for i, f in enumerate(ids):
        both = out["views"][i]["hit"] & (s["depth"][f] > 0)
        assert both.sum() > 0.9 * (s["depth"][f] > 0).sum()
        dz = np.abs(out["depth"][i][both] - s["depth"][f][both])
        dl = np.abs(out["intensity"][i][both] - s["lum"][f][both])
        print(f, both.sum(), dz.mean() / vs, dz.max() / vs, dl.mean(), np.median(dl))
        # measured (views 0, 3): mean |dz| 0.043 / 0.043 voxel, max 0.27 / 0.27 voxel; mean |dI| 0.0060 / 0.0041, median 0.0023 / 0.0017
        assert dz.mean() <= 0.08 * vs and dz.max() <= 0.4 * vs
        assert dl.mean() <= 0.01 and np.median(dl) <= 0.004


def test_distortion_round_trip():
    """With lens distortion, the hit point projected through observation_weight's forward model lands on the pixel centre."""
    s = _truth_scene()
    g = dict(xyz=s["xyz"], sdf0=s["sdf0"], sdf_refined=s["sdf_true"], albedo=s["albedo"], weight=s["weight"], voxel_size=s["voxel_size"])
    grid = rr.grid_of(g, "refined")
    dist = np.array([0.12, -0.05, 0.01, 0.002, -0.003])
    cam = rr.camera(s["intr"], dist)
    rt = rr.pose_rt(s["poses_true"])[1]
    _, H, W = s["depth"].shape
    v = rr.render_view(grid, rt, cam, W, H, photometric=False)
    o, dn = v["ray"]
    hit = v["hit"]
    p = o[None, :] + v["s_hit"][hit][:, None] * dn[hit]
    pu, pv = rr.project(p, rt, cam)
    vv, uu = np.nonzero(hit)
    err = np.maximum(np.abs(pu - uu), np.abs(pv - vv)).max()
    # measured: 1.9e-5 px over 6376 hit pixels (float rounding of the fixed-point undistortion and of the projection)
    assert hit.sum() > 1000 and err <= 2e-4, err


def test_golden_fixture():
    """The restatement reproduces the pinned fixture (the device renderer is checked against the same file on the GPU)."""
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden_render as mg
    gold = np.load(os.path.join(HERE, "golden", "tiny_render.npz"))
    out = mg.compute()
    for k, v in out.items():
        assert v.shape == gold[k].shape and v.tobytes() == gold[k].tobytes(), k
