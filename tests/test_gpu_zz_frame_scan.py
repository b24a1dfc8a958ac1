"""The two frame scans, the observation selection (k_select_obs) and the recolouring (k_recolor), where the bounds of their conservative
frame culling (i3d_observe.cuh: k_depth_tiles, frame_may_see, frame_candidates) are tight: NaN and +-inf depth with the occlusion test
off and on, strong lens distortion that folds the image, cameras against or inside the surface, partial tiles and principal points
outside the image, pyramid levels, depth on the edges of the occlusion band, frame counts around the 32-frame mask words and the
512-frame limit of the culling, non-finite poses and partial warps.

Every case runs the engine in two child processes (the culling switches are read once per process): one with I3D_CULL_STATS=1, whose
selection, E_g row set and recoloured colours must be bit-equal to the oracle's, and one with I3D_NO_CULL=1, whose outputs must be
byte-equal to the first.  The first child's culling statistics show that the case reaches the culling: some (warp, frame) pairs are
skipped and some visited.  The recolouring has no statistics of its own; it scans the same geometry as the selection."""
import functools
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from intrinsic3d_b200.ctypes_defs import default_params
from intrinsic3d_b200.engine import Engine
a = json.loads(sys.argv[2])
z = np.load(a["scene"])
s = {k: z[k] for k in z.files}
s["pyr_scale"] = float(s["pyr_scale"])
p = default_params()
p.thres_shell, p.occlusion_distance, p.num_observations, p.build_only = a["thres_shell"], a["occlusion"], a["K"], 1
e = Engine(0)
e.load_scene(s)
e.gn_iteration(p)
fr, w, act = e.debug_observations(a["Kobs"])
rows = e.debug_rows(want_jac=False)
out = dict(frames=fr, weights=w, active=act, row_voxel=rows["voxel"], row_frame=rows["frame"])
if a["recolor_K"] >= 0:
    e2 = Engine(0)
    e2.load_scene(s)
    e2.upload_color_frames(s["color"])
    out["recolor_counts"] = np.array(e2.recompute_colors(a["occlusion"], a["recolor_K"]), np.int64)
    out["colors"] = e2.download_colors()
np.savez(a["out"], **out)
"""


def _child(tmp_path, tag, scene_file, args, env_on):
    env = dict(os.environ)
    for k in ("I3D_NO_CULL", "I3D_CULL_STATS"):
        env.pop(k, None)
    env[env_on] = "1"
    out = str(tmp_path / f"{tag}.npz")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT, json.dumps(dict(args, scene=scene_file, out=out))]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    z = np.load(out)
    return {k: z[k] for k in z.files}, r.stderr


def _rows(voxel, frame):
    return sorted((int(v), int(f)) for v, f in zip(voxel, frame) if f >= 0)


def check_case(tmp_path, s, K=5, occlusion=0.02, recolor=True, culls=True):
    """Engine (culled and unculled, in child processes) against the oracle on scene s; returns (visited, total) of the culled run"""
    import oracle
    from intrinsic3d_b200.ctypes_defs import default_params
    from intrinsic3d_b200.scene import make_color_frames
    t0 = time.time()
    F = s["poses"].shape[0]
    Kobs = K if 0 < K <= F else F
    recolor_K = min(K, 8) if recolor else -1
    s = dict(s)
    s["color"] = make_color_frames(s)
    scene_file = str(tmp_path / "scene.npz")
    np.savez(scene_file, **{k: np.asarray(v) for k, v in s.items()})
    args = dict(thres_shell=float(s["thres_shell"]), occlusion=float(occlusion), K=int(K), Kobs=int(Kobs), recolor_K=int(recolor_K))
    got, err = _child(tmp_path, "cull", scene_file, args, "I3D_CULL_STATS")
    ref, _ = _child(tmp_path, "nocull", scene_file, args, "I3D_NO_CULL")
    # the culled run is byte-equal to the unculled one
    assert got.keys() == ref.keys()
    for k in got:
        assert got[k].tobytes() == ref[k].tobytes(), k
    # and bit-equal to the oracle
    p = default_params()
    p.thres_shell, p.occlusion_distance, p.num_observations, p.build_only = float(s["thres_shell"]), float(occlusion), int(K), 1
    o = oracle.Oracle(threads=min(32, os.cpu_count() or 8))
    o.load_scene(s)
    o.gn_iteration(p)
    fo, wo, ao = o.observations(Kobs)
    assert np.array_equal(got["active"], ao)
    bad = np.nonzero((got["frames"] != fo).any(1))[0]
    assert len(bad) == 0, dict(voxels=len(bad), first=[(int(v), got["frames"][v].tolist(), fo[v].tolist()) for v in bad[:5]])
    assert np.array_equal(got["weights"].view(np.uint32), wo.view(np.uint32))
    ro = o.rows(0)
    assert _rows(got["row_voxel"], got["row_frame"]) == _rows(ro["voxel"], ro["aux"])
    if recolor:
        o2 = oracle.Oracle(threads=min(32, os.cpu_count() or 8))
        o2.load_scene(s)
        o2.set_color_frames(s["color"])
        assert tuple(got["recolor_counts"].tolist()) == o2.recompute_colors(float(occlusion), recolor_K)
        assert np.array_equal(got["colors"], o2.colors())
    m = re.search(r"frame culling: (\d+) of (\d+)", err)
    assert m, err[-2000:]
    visited, total = int(m.group(1)), int(m.group(2))
    assert 0 < visited and total > 0
    if culls:
        assert visited < total, (visited, total)
    print(f"frame scan: F={F} K={K} occ={occlusion} active={int(ao.sum())} observations={int((fo >= 0).sum())} "
          f"visited {visited} of {total} ({100.0 * visited / total:.1f} %), {time.time() - t0:.1f} s")
    return visited, total


@functools.lru_cache(maxsize=None)
def _scene(name="tiny", **kw):
    from intrinsic3d_b200.scene import config_scene
    return config_scene(name, **kw)


def _base(name="tiny", **kw):
    s = _scene(name, **kw)
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in s.items()}


def _aside(s, f):
    """moves frame f 2 m back and gives it no depth: a frame every warp can drop, whatever the footprint bound of its camera"""
    s["poses"][f, 5] += 2.0
    s["depth"][f] = 0.0
    return s


def _nan_depth(s):
    """frame 0 entirely NaN (a dropped frame), frame 1 NaN in 32x32 blocks, frame 2 scattered NaN pixels, frame 3 NaN mixed with 0"""
    rng = np.random.default_rng(4)
    d = s["depth"]
    F, H, W = d.shape
    d[0] = np.nan
    for y in range(0, H, 64):
        for x in range(16, W, 64):
            d[1, y:y + 32, x:x + 32] = np.nan
    d[2][rng.random((H, W)) < 0.1] = np.nan
    d[3][rng.random((H, W)) < 0.5] = np.nan
    d[3][rng.random((H, W)) < 0.3] = 0.0
    return s


@pytest.mark.parametrize("occlusion", [0.0, -1.0])
def test_nan_depth_without_occlusion_test(occlusion, tmp_path):
    """The occlusion test off: the reference observes a NaN depth (it rejects d <= 0 only), so a frame that is NaN under a warp's
    footprint must not be culled"""
    check_case(tmp_path, _aside(_nan_depth(_base()), 5), occlusion=occlusion)


def test_nan_and_inf_depth_with_occlusion_test(tmp_path):
    """The occlusion test on: NaN and +-inf depths are rejected by the reference, and the culling may drop tiles made of them"""
    s = _nan_depth(_base())
    rng = np.random.default_rng(5)
    r = rng.random(s["depth"][4].shape)
    s["depth"][4][r < 0.2] = np.inf
    s["depth"][4][(r >= 0.2) & (r < 0.4)] = -np.inf
    s["depth"][5, :, : s["depth"].shape[2] // 2] = np.inf
    check_case(tmp_path, s, occlusion=0.02)


DIST = {"k1-0.4": [-0.4, 0.12, -0.02, 0.01, -0.01], "k1+0.3": [0.3, -0.08, 0.02, -0.01, 0.01]}


@pytest.mark.parametrize("dist", list(DIST))
@pytest.mark.parametrize("occlusion", [0.02, 10.0])
def test_strong_distortion(dist, occlusion, tmp_path):
    """k1 = -0.4 / +0.3 with k2, k3, p1, p2 != 0 (d = k1, k2, k3, p1, p2) and the cameras moved in to 0.7 of their distance so that the
    object fills most of the image: the Lipschitz bound of the distortion and the distorted centre.  The depth is the undistorted rendering (any depth must be
    culled exactly); occlusion 10 m lets every in-image pixel of positive depth through, so the footprint bound alone decides"""
    s = _base()
    s["dist"] = np.array(DIST[dist], np.float64)
    s["poses"][:, 3:] *= 0.7
    check_case(tmp_path, _aside(s, 5), occlusion=occlusion)


def test_distortion_folds_inside_footprints(tmp_path):
    """A wide camera (fx = 30 px on 160 x 120) with k1 = -0.4, moved sideways so that the object sits near r = 1.6: the radial factor
    1 + k1 r^2 is negative beyond r = 1.58, inside the warps' footprints, so the distortion map folds there"""
    s = _base()
    s["dist"] = np.array([-0.4, 0.0, 0.0, 0.01, 0.01], np.float64)
    s["intr"] = np.array([30.0, 30.0, 79.5, 59.5])
    s["poses"][:, 3] += 0.2
    check_case(tmp_path, _aside(s, 5), occlusion=10.0)


@pytest.mark.parametrize("occlusion", [0.02, 0.0])
def test_cameras_at_and_inside_the_surface(occlusion, tmp_path):
    """Frame 0 three voxels in front of the surface, frame 1 at the object's centre looking out (the voxels behind it have z < 0),
    frame 2 with its camera plane through the object: zmin near 1e-3 and below, huge footprints.  The depth of frame 1 is the object's
    radius so that the voxels in front of it pass the occlusion test"""
    s = _base()
    vs = float(s["voxel_size"])
    rho = 10.0 * vs
    s["poses"][0] = [0, 0, 0, 0, 0, rho + 3 * vs]
    s["poses"][1] = [0, 0, 0, 0, 0, 0]
    s["poses"][2] = [0, 0, 0, 0, 0, 1e-3]
    s["depth"][1] = np.float32(rho)
    s["depth"][2] = np.float32(0.02)
    check_case(tmp_path, _aside(s, 5), occlusion=occlusion, culls=occlusion > 0)


def _crop(s, x0, y0, W, H):
    s["depth"] = np.ascontiguousarray(s["depth"][:, y0:y0 + H, x0:x0 + W])
    s["lum"] = np.ascontiguousarray(s["lum"][:, y0:y0 + H, x0:x0 + W])
    s["intr"] = s["intr"] - np.array([0, 0, x0, y0])
    return s


@pytest.mark.parametrize("crop", [(0, 0, 100, 75), (50, 30, 100, 75), (120, 40, 100, 75), (80, 60, 33, 31), (100, 75, 33, 31)],
                         ids=["100x75", "100x75_offcentre", "100x75_pp_outside", "33x31", "33x31_pp_outside"])
def test_partial_tiles_and_principal_point(crop, tmp_path):
    """W x H not a multiple of 32, crops of a 200 x 150 rendering whose principal point moves off-centre and outside the image: partial
    tiles, the +2 px margin, the entirely-outside test and the clamping of the tile range"""
    x0, y0, W, H = crop
    s = _crop(_base(width=200, height=150), x0, y0, W, H)
    check_case(tmp_path, s, occlusion=0.02)


@pytest.mark.parametrize("level", [1, 2])
def test_pyramid_levels(level, tmp_path):
    """Frames of pyramid level 1 and 2 (pyr_scale 0.5, 0.25: the intrinsics scaled in the scan) of 160 x 120, subsampled"""
    s = _base()
    k = 1 << level
    s["depth"] = np.ascontiguousarray(s["depth"][:, ::k, ::k])
    s["lum"] = np.ascontiguousarray(s["lum"][:, ::k, ::k])
    s["pyr_scale"] = 1.0 / k
    check_case(tmp_path, s, occlusion=0.02)


@pytest.mark.parametrize("occlusion", [1e-6, 0.02, 10.0])
def test_depth_on_the_occlusion_edges(occlusion, tmp_path):
    """The rendered depth moved by +occ(1 + 1e-6), -occ(1 - 1e-6), -occ(1 + 1e-6), +occ(1 - 1e-6) and by the floats next to +-occ:
    the iso-points sit on the edges of the occlusion band, where the tolerance 1.001 occ + 1e-4 of the culling is tight"""
    s = _base()
    o = np.float32(occlusion)
    up, dn = np.nextafter(o, np.float32(np.inf)), np.nextafter(o, np.float32(0))
    shifts = [o * np.float32(1 + 1e-6), -o * np.float32(1 - 1e-6), -o * np.float32(1 + 1e-6), o * np.float32(1 - 1e-6), up, -dn]
    d = s["depth"]
    for f in range(d.shape[0]):
        hit = d[f] > 0
        d[f][hit] = d[f][hit] + shifts[f % len(shifts)]
    check_case(tmp_path, s, occlusion=occlusion, culls=occlusion < 1.0)


@pytest.mark.parametrize("F,K", [(31, 5), (32, 8), (33, 1), (512, 5), (513, 8)])
def test_frame_counts(F, K, tmp_path):
    """Frame counts around the 32-frame mask words and the 512-frame limit of the culling (513 frames take the unculled path, which
    counts 32 visits per mask word: 17 words, 544 visits per warp against 513 frames), k_select_obs / k_recolor <5> and <8>"""
    s = _base(frames=F, width=64, height=48)
    v, t = check_case(tmp_path, s, K=K, occlusion=0.02, culls=F <= 512)
    if F > 512:
        assert v >= t and v * 513 == t * 544


def test_more_observations_than_frames(tmp_path):
    """K = 8 on 6 frames: every frame a candidate of the top-K"""
    check_case(tmp_path, _base(), K=8, occlusion=0.02)


def test_non_finite_poses(tmp_path):
    """NaN and inf in two frames' poses (set on both sides): a non-finite frame centre is never culled; the other frames still are"""
    s = _base()
    s["poses"][2, 3] = np.nan
    s["poses"][4, 0] = np.inf
    check_case(tmp_path, s, occlusion=0.02)


@pytest.mark.parametrize("n_active", [1, 31, 33])
def test_few_active_voxels(n_active, tmp_path):
    """1, 31 and 33 active voxels: idle lanes in the warps' bounding spheres"""
    from intrinsic3d_b200.ctypes_defs import default_params
    from test_gpu_normal_equations import _active_cut
    s = _base()
    p = default_params()
    p.thres_shell = s["thres_shell"]
    s["thres_shell"] = _active_cut(s, n_active, p)
    check_case(tmp_path, _aside(s, 5), occlusion=0.02, recolor=False)


def test_incoherent_voxel_order(tmp_path):
    """Voxels in raster order instead of bricks: warps span long rows of the object, with large bounding spheres"""
    check_case(tmp_path, _base(brick_order=False), occlusion=0.02)
