"""The device stages around the refinement core against their references at the size the product runs them: the C2 scene (~500 K
voxels, 50 frames at 640 x 480) and, for the mesh, C3.  Each case keeps the bar of its small-scale test (tests/test_gpu_zz_fusion.py,
_gridops, _recolor, _lighting, _mesh, _render, _track, _track_color) and asserts that the mechanism only this size reaches was reached:
the fusion hash table near 1 M entries and growing under load, an upsample to ~4 M voxels, more than 1024 lighting subvolumes, the
mesh union-find and welding at a few hundred thousand faces, the renderer's brick skipping on a 0.5 M-voxel grid, 1200 tracking
tiles per frame.  Every case prints those counts, the device time of the stage and the CPU time of its reference."""
import os
import time

import numpy as np
import pytest

import render_ref as rr
import track_color_ref as tc
import track_ref as tr
from fusion_ref import scene_inputs
from test_gpu_zz_fusion import _fuse_engine, _oracle, _params as _fusion_params, _same
from test_gpu_zz_gridops import _same_grid
from test_gpu_zz_lighting import _compare as _lighting_compare, _lighting_params
from test_gpu_zz_mesh import COUNTS, _check as _mesh_check, _check_all as _mesh_check_all, _engine_with
from test_gpu_zz_render import _check as _render_check, _skip_same
from test_gpu_zz_track import _compare as _track_compare, _dcam, _initial_same
from test_gpu_zz_track import _rel
from test_odometry import live_grid

pytestmark = pytest.mark.gpu
THREADS = os.cpu_count()
TRACK_IDS = [7, 32]                         # two frames of the orbit, away from its start
RENDER_IDS = [3, 28]
DISTORTION = np.array([0.1, -0.04, 0.01, 0.002, -0.003])
# the synthetic colour frames are smooth at 640 x 480: the default gradient gate (0.01 per pixel) keeps ~5 K photometric rows per frame,
# 0.002 keeps ~20 K
PHOTO = dict(min_color_gradient=0.002)
FUSION_INTEGRATE = ("fusion_prep", "fusion_alloc", "fusion_integrate")
LIGHTING = ("light_subvolumes", "light_accumulate", "light_solve", "light_interpolate")


def _report(case, **kw):
    print(f"scale case {case}: " + ", ".join(f"{k} {round(v, 3) if isinstance(v, float) else v}" for k, v in kw.items()))


def _ms(e, *phases):
    return sum(e.phase_ms(p) for p in phases)


class _Clock:
    def __enter__(self):
        self.t = time.perf_counter()
        return self

    def __exit__(self, *exc):
        self.s = time.perf_counter() - self.t


@pytest.fixture(scope="module")
def c2():
    from intrinsic3d_b200.scene import config_scene
    return config_scene("c2", device="cuda")


@pytest.fixture(scope="module")
def fusion_ref(c2):
    """the float oracle's fusion of all 50 C2 frames, before and after finish(1) (correctSDF as Jacobi sweeps)"""
    p = _fusion_params(c2)
    inp = scene_inputs(c2)
    o = _oracle(p)
    with _Clock() as ci:
        assert o.integrate(*inp) == 0
    vol = o.volume()
    with _Clock() as cf:
        sweeps = o.finish(1)
    return dict(p=p, inp=inp, volume=vol, finished=o.volume(), sweeps=sweeps, cpu_integrate=ci.s, cpu_finish=cf.s)


def _store_engine(c2, p):
    """an engine with the 50 C2 frames in its sensor store, all integrated from the store at their true poses with fusion params p"""
    from intrinsic3d_b200.engine import Engine
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(c2)
    e = Engine(0)
    e.sensor_frames_begin(dcam, ccam, depth.shape[0])
    e.sensor_frames_add(depth, bgr)
    e.fusion_begin(p)
    e.fusion_integrate_sensor(np.arange(depth.shape[0]), c2w, w2c)
    return e


@pytest.fixture(scope="module")
def sensor_fusion(c2, fusion_ref):
    """the fusion from the sensor store, still in progress"""
    e = _store_engine(c2, fusion_ref["p"])
    yield e
    e.close()


@pytest.fixture(scope="module")
def finished(c2, fusion_ref):
    """the fusion from the sensor store, finished: the engine's grid is the fused C2 grid"""
    e = _store_engine(c2, fusion_ref["p"])
    m = e.fusion_finish()
    yield e, m
    e.close()


def _oracle_of(s):
    import oracle
    o = oracle.Oracle(threads=THREADS)
    o.load_scene(s)
    return o


def _scene_engine(s):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(s)
    return e


# ---- 1-4: fusion --------------------------------------------------------------------------------------------------------------------
def test_c2_fusion_host_frames_bit_exact(fusion_ref):
    vo = fusion_ref["volume"]
    e = _fuse_engine(fusion_ref["p"], fusion_ref["inp"])
    _same(e.fusion_volume(), vo)
    assert len(vo["xyz"]) > 900_000
    _report(1, entries=len(vo["xyz"]), integrated=int((vo["weight"] > 0).sum()), growths=e.phase_count("fusion_growths"),
            device_ms=_ms(e, *FUSION_INTEGRATE), cpu_s=fusion_ref["cpu_integrate"])
    e.close()


def test_c2_fusion_from_sensor_store_same_bytes(fusion_ref, sensor_fusion):
    _same(sensor_fusion.fusion_volume(), fusion_ref["volume"])
    _report(2, entries=len(fusion_ref["volume"]["xyz"]), device_ms=_ms(sensor_fusion, *FUSION_INTEGRATE))


# A full table grows to at least twice its slots, then on until it is at most a quarter full; the inserts of the threads still running when
# it fills count too, so one growth can double more than once: from 2^18 slots the 952 K entries (2^21 slots) take two growths, from 2^16
# at least three.
@pytest.mark.parametrize("cap,growths", [(1 << 18, 2), (1 << 16, 3)])
def test_c2_fusion_growth_under_load_same_bytes(c2, fusion_ref, cap, growths):
    e = _fuse_engine(_fusion_params(c2, cap=cap), fusion_ref["inp"])
    got = e.phase_count("fusion_growths")
    assert got >= growths
    _same(e.fusion_volume(), fusion_ref["volume"])
    _report(3, initial_slots=cap, growths=got, entries=len(fusion_ref["volume"]["xyz"]), device_ms=_ms(e, *FUSION_INTEGRATE))
    e.close()


def test_c2_fusion_finish_bit_exact_against_jacobi_oracle(fusion_ref, finished):
    e, m = finished
    vj = fusion_ref["finished"]
    g = e.download_grid()
    assert m == len(vj["xyz"]) > 700_000
    assert np.array_equal(g["xyz"], vj["xyz"])
    assert np.array_equal(g["sdf0"], vj["sdf"].astype(np.float64)) and np.array_equal(g["sdf_refined"], g["sdf0"])
    assert np.array_equal(g["weight"].view(np.uint32), vj["weight"].view(np.uint32)) and np.array_equal(g["rgb"], vj["rgb"])
    assert (g["albedo"] == 0.6).all() and (g["weight"] > 0).all()
    assert g["voxel_size"] == np.float32(fusion_ref["p"].voxel_size)
    assert e.phase_count("fusion_sweeps") == fusion_ref["sweeps"]
    _report(4, voxels=m, sweeps=fusion_ref["sweeps"], device_ms=_ms(e, "fusion_correct", "fusion_finish"), cpu_s=fusion_ref["cpu_finish"])


# ---- 5: prune, upsample to ~4 M voxels, and the residual build on the rebuilt tables ------------------------------------------------
def test_c2_prune_upsample_and_residual_build_bit_exact(c2):
    import ctypes as C
    from intrinsic3d_b200.ctypes_defs import default_params
    e, o = _scene_engine(c2), _oracle_of(c2)
    shell = float(c2["thres_shell"])
    with _Clock() as cp:
        pruned = o.clear_voxels_outside_thin_shell(shell)
    assert e.clear_voxels_outside_thin_shell(shell) == pruned and 0 < pruned < len(c2["xyz"])
    t_prune = e.phase_ms("prune")
    _same_grid(e, o)
    with _Clock() as cu:
        mo = o.upsample_grid()
    assert e.upsample_grid() == mo == 8 * pruned
    t_up = e.phase_ms("upsample")
    _same_grid(e, o)
    assert mo > 3_900_000
    # the upsample drops the per-voxel SH on both sides: the same constant SH everywhere again
    sh = np.ascontiguousarray(np.tile(c2["sh"][0], (mo, 1)), np.float64)
    e.set_sh(sh)
    o._check(o.L.i3do_set_sh(o.h, sh.ctypes.data_as(C.POINTER(C.c_double))))
    p = default_params()
    p.thres_shell = shell
    p.build_only = 1
    je = e.gn_iteration(p)
    with _Clock() as cg:
        jo = o.gn_iteration(p)
    assert list(je.type_residuals) == list(jo.type_residuals) and jo.type_residuals[0] > 100_000
    np.testing.assert_allclose(list(je.type_sum_weights), list(jo.type_sum_weights), rtol=1e-9)
    np.testing.assert_allclose(je.cost_initial, jo.cost_initial, rtol=1e-9)
    fe, we, ae = e.debug_observations(5)
    fo, wo, ao = o.observations(5)
    assert np.array_equal(ae, ao) and np.array_equal(fe, fo) and np.array_equal(we.view(np.uint32), wo.view(np.uint32))
    _report(5, pruned=pruned, upsampled=mo, residuals=list(jo.type_residuals), device_ms_prune=t_prune,
            device_ms_upsample=t_up, cpu_s_prune=cp.s, cpu_s_upsample=cu.s, cpu_s_build=cg.s)
    e.close()


# ---- 6: recolouring from 50 colour frames ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def c2_colors(c2):
    from intrinsic3d_b200.scene import make_color_frames
    return make_color_frames(c2)


@pytest.mark.parametrize("K", [5, 8])
def test_c2_recolor_bit_exact(c2, c2_colors, K):
    e, o = _scene_engine(c2), _oracle_of(c2)
    e.upload_color_frames(c2_colors)
    o.set_color_frames(c2_colors)
    ce = e.recompute_colors(0.02, K)
    with _Clock() as cc:
        co = o.recompute_colors(0.02, K)
    assert ce == co and co[1] > 2 * co[0]
    rgb_e, rgb_o = e.download_colors(), o.colors()
    assert np.array_equal(rgb_e, rgb_o)
    assert (rgb_o != c2["rgb"]).any(1).sum() > 0.9 * co[0]
    assert co[0] > 300_000
    _report(6, K=K, recoloured=co[0], observations=co[1], device_ms=e.phase_ms("recolor"), cpu_s=cc.s)
    e.close()


# ---- 7: lighting with more than 1024 subvolumes ------------------------------------------------------------------------------------
def _lighting_pair(c2, **kw):
    from intrinsic3d_b200 import engine
    import oracle
    e, o = _scene_engine(c2), _oracle_of(c2)
    ie = e.estimate_lighting(_lighting_params(engine, c2, **kw))
    with _Clock() as cl:
        io = o.estimate_lighting(_lighting_params(oracle, c2, **kw))
    return e, o, ie, io, cl.s


@pytest.mark.parametrize("size", [0.02, 0.01])
def test_c2_lighting_many_subvolumes(c2, size):
    e, o, ie, io, cpu = _lighting_pair(c2, subvolume_size=size)
    assert io.num_subvolumes > 1024
    _report(7, subvolume_size=size, subvolumes=io.num_subvolumes, data_rows=io.num_data_rows, lm=(ie.lm_iterations, io.lm_iterations),
            cg=(ie.cg_iterations_total, io.cg_iterations_total), device_ms=_ms(e, *LIGHTING), cpu_s=cpu)
    _lighting_compare(e, o, ie, io)
    e.close()


@pytest.mark.parametrize("size", [0.02, 0.01])
def test_c2_lighting_many_subvolumes_fixed_cg(c2, size):
    """30 CG iterations in each of 2 LM iterations on both sides: the SH without the CG stopping rule"""
    e, o, ie, io, cpu = _lighting_pair(c2, subvolume_size=size, min_linear_solver_iterations=30, max_linear_solver_iterations=30,
                                       max_iterations=2)
    idx_e, sh_e = e.download_lighting()
    idx_o, sh_o = o.lighting()
    assert np.array_equal(idx_e, idx_o) and len(idx_o) > 1024
    assert (ie.num_subvolumes, ie.num_data_rows, ie.num_reg_pairs, ie.lm_iterations, ie.num_successful_steps, ie.cg_iterations_total) == \
           (io.num_subvolumes, io.num_data_rows, io.num_reg_pairs, io.lm_iterations, io.num_successful_steps, io.cg_iterations_total)
    ref = np.abs(sh_o).max()
    assert np.abs(sh_e - sh_o).max() <= 1e-8 * ref
    vsh_e, has_e = e.download_voxel_sh()
    vsh_o, has_o = o.voxel_sh()
    assert np.array_equal(has_e, has_o) and np.abs(vsh_e - vsh_o).max() <= 1e-8 * ref
    _report("7b", subvolume_size=size, subvolumes=io.num_subvolumes, cg=io.cg_iterations_total, device_ms=_ms(e, *LIGHTING), cpu_s=cpu)
    e.close()


# ---- 8-10: mesh extraction: welding over ~10^6 corner keys and the union-find of the largest-component filter --------------------
def _mesh_ms(m):
    i = m["info"]
    return i.ms_classify + i.ms_emit + i.ms_weld + i.ms_clean + i.ms_components


def _counts(m):
    return {k: int(getattr(m["info"], k)) for k in COUNTS}


def test_c2_mesh_bytes_equal(c2):
    e = _scene_engine(c2)
    with _Clock() as cm:
        ms = _mesh_check_all(e)                       # fused and refined, each with the filter off and on
    assert ms[3]["info"].num_faces > 200_000
    for m, name in zip(ms, ("fused", "fused largest", "refined", "refined largest")):
        _report(8, mesh=name, device_ms=_mesh_ms(m), **_counts(m))
    _report(8, cpu_s_all_four=cm.s)
    e.close()


def _face_components(faces, V):
    """the number of face-connected components (faces sharing a vertex are connected), as mesh_ref.largest_component counts them"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    r = np.concatenate([faces[:, 0], faces[:, 0]])
    c = np.concatenate([faces[:, 1], faces[:, 2]])
    _, lab = connected_components(coo_matrix((np.ones(len(r)), (r, c)), shape=(V, V)), directed=False)
    return len(np.unique(lab[faces[:, 0]]))


def test_c2_noisy_mesh_many_components_bytes_equal(c2):
    """the construction of test_gpu_zz_mesh.py::test_many_components_bytes_equal at C2: a noisy refined sdf scatters the surface"""
    vs = float(c2["voxel_size"])
    noisy = c2["sdf0"] + np.random.default_rng(4).normal(0.0, 1.5 * vs, len(c2["sdf0"]))
    e = _engine_with(c2["xyz"], c2["sdf0"], noisy, c2["weight"], c2["rgb"], vs)
    with _Clock() as cm:
        full, largest = _mesh_check_all(e, sources=("refined",))
    comps = _face_components(full["faces"], len(full["vertices"]))    # byte-equal to the reference mesh
    assert largest["info"].num_faces < largest["info"].num_faces_clean
    assert comps > 1000
    _report(9, components=comps, device_ms=_mesh_ms(largest), cpu_s_both=cm.s, **_counts(largest))
    e.close()


def test_c3_refined_mesh_largest_component_bytes_equal():
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c3", device="cuda")
    e = _scene_engine(s)
    g = e.download_grid()
    with _Clock() as cm:
        m = _mesh_check(e, g, "refined", True)
    assert m["info"].num_faces > 800_000
    _report(10, voxels=len(g["xyz"]), device_ms=_mesh_ms(m), cpu_s=cm.s, **_counts(m))
    e.close()


# ---- 11: keyframe render at 640 x 480 over the brick bitmap of a 0.5 M-voxel grid --------------------------------------------------
def test_c2_render_bytes_equal(c2):
    e = _scene_engine(c2)
    for src, ids in (("refined", RENDER_IDS), ("fused", RENDER_IDS[:1])):      # one fused view: the march is the same, only the sdf differs
        with _Clock() as cr:
            out, _ = _render_check(e, ids, src)
        ms = e.phase_ms("render")
        assert all(st["num_hit"] > 90_000 for st in out["stats"]), out["stats"]
        na, nb = _skip_same(e, ids, src)
        assert na < nb
        _report(11, source=src, views=ids, hits=[st["num_hit"] for st in out["stats"]], samples_skip=na, samples_dense=nb,
                device_ms=ms, cpu_s=cr.s)
    e.set_camera(c2["poses"], c2["intr"], DISTORTION)
    with _Clock() as cr:
        out, _ = _render_check(e, RENDER_IDS[:1])
    ms = e.phase_ms("render")
    assert out["stats"][0]["num_hit"] > 90_000, out["stats"]
    na, nb = _skip_same(e, RENDER_IDS[:1])
    assert na < nb
    _report(11, source="refined, distorted", views=RENDER_IDS[:1], hits=out["stats"][0]["num_hit"], samples_skip=na, samples_dense=nb,
            device_ms=ms, cpu_s=cr.s)
    e.close()


# ---- 12-13: tracking at 640 x 480: 1200 tiles per frame at level 0 -----------------------------------------------------------------
def _tiles(plane):
    H, W = plane.shape[-2:]
    return -(-H // tr.TILE) * -(-W // tr.TILE)


def test_c2_track_against_finished_fusion(c2, finished):
    e, _ = finished
    g = e.download_grid()
    grid = rr.Grid(g["xyz"], g["sdf0"], g["albedo"], g["weight"], g["voxel_size"])
    dcam = _dcam(c2)
    depth = c2["depth"]
    start = tr.perturb(tr.aa_to_rt(c2["poses_true"])[TRACK_IDS], 0.5, 0.005, seed=12)
    # the input pose's prediction planes and level-0 systems on every level, no update
    out = e.track_sensor_frames(TRACK_IDS, start, "fused", num_levels=3, iterations=(0, 0, 0))
    ms = e.phase_ms("track")
    with _Clock() as cr:
        frames = [tr.Frame(depth[f], start[k], dcam, tr.params(num_levels=3, iterations=(0, 0, 0)), grid=grid).run()
                  for k, f in enumerate(TRACK_IDS)]
    _track_compare(e, frames, TRACK_IDS, out, 3)
    assert np.array_equal(out[0], start)
    for info, f in zip(out[1], frames):
        _initial_same(info, f)
    tiles = _tiles(e.debug_track_planes(0, len(TRACK_IDS))["depth"])
    corr = [i["correspondences"] for i in out[1]]
    assert tiles == 1200 and min(corr) > 50_000
    _report(12, schedule="(0,0,0)", tiles_level0=tiles, correspondences=corr, device_ms=ms, cpu_s=cr.s)
    # the restated frames reuse the prediction at the input pose from here on
    pred = [(f.pdepth, f.pnrm) for f in frames]

    def restate(**over):
        p = tr.params(**over)
        return [tr.Frame(depth[f], start[k], dcam, p, prediction=pred[k]).run() for k, f in enumerate(TRACK_IDS)]
    out = e.track_sensor_frames(TRACK_IDS, start, "fused", num_levels=1, iterations=(1,))
    ms = e.phase_ms("track")
    with _Clock() as cr:
        frames = restate(num_levels=1, iterations=(1,))
    _track_compare(e, frames, TRACK_IDS, out, 1)
    assert all(i["iterations"] == 1 and i["status"] == 0 for i in out[1])
    _report(12, schedule="(1,)", correspondences=[i["correspondences"] for i in out[1]], device_ms=ms, cpu_s=cr.s)
    out = e.track_sensor_frames(TRACK_IDS, start, "fused")
    ms = e.phase_ms("track")
    with _Clock() as cr:
        frames = restate()
    _track_compare(e, frames, TRACK_IDS, out, 3, planes=False, pose_tol=1e-6)
    assert all(i["status"] == 0 for i in out[1])
    r, t = tr.pose_errors(out[0], tr.aa_to_rt(c2["poses_true"])[TRACK_IDS])
    _report(12, schedule="default", iterations=[i["iterations"] for i in out[1]], correspondences=[i["correspondences"] for i in out[1]],
            rot_deg=float(r.max()), centre_mm=float(1e3 * t.max()), device_ms=ms, cpu_s=cr.s)


def _check_rgbd_against_restatement(e, s, ids, start, levels, iterations, color):
    """test_gpu_zz_track_color.py's _check_against_restatement with colour parameters other than the defaults, on both sides"""
    dcam, depth, ccam, bgr, _, _ = scene_inputs(s)
    v = e.fusion_volume()
    keep = v["weight"] > 0
    grid = live_grid(v, np.float32(s["voxel_size"]))
    inten = {f: tc.frame_intensity(bgr[f], ccam, dcam) for f in ids}
    out = e.fusion_track_sensor_frames_rgbd(ids, start, color=color, num_levels=levels, iterations=iterations)
    p = tr.params(num_levels=levels, iterations=iterations)
    c = tc.color_params(**color)
    frames = [tc.ColorFrame(depth[f], inten[f], start[k], dcam, p, c, grid=grid, rgb=v["rgb"][keep]).run() for k, f in enumerate(ids)]
    n = len(ids)
    sums, T = e.debug_track_system(n)
    csum = e.debug_track_color_system(n)
    for k, f in enumerate(frames):
        info = out[1][k]
        assert [f.status, f.iterations, f.correspondences] == [info["status"], info["iterations"], info["correspondences"]], k
        assert f.sys[28] == sums[k, 28] and _rel(sums[k], f.sys), (k, sums[k], f.sys)
        assert f.sys_c[28] == csum[k, 28] and _rel(csum[k], f.sys_c), (k, csum[k], f.sys_c)
        assert [f.first[0], f.last[0]] == [info["color"]["first_rows"], info["color"]["last_rows"]]
        assert np.abs(np.array(f.w2c) - out[0][k]).max() <= 1e-12 and np.abs(np.array(f.T) - T[k]).max() <= 1e-12
    for l in range(levels):
        P = e.debug_track_color_planes(l, n)
        for k, f in enumerate(frames):
            assert P["intensity"][k].tobytes() == f.inten[l].tobytes(), ("intensity", l, k)
            assert P["grad_x"][k].tobytes() == f.grads[l][0].tobytes() and P["grad_y"][k].tobytes() == f.grads[l][1].tobytes(), (l, k)
            if l == 0:
                assert P["model_intensity"][k].tobytes() == f.pint.tobytes(), ("model_intensity", k)
    return out, frames


def test_c2_track_rgbd_against_fusion_in_progress(c2, sensor_fusion):
    e = sensor_fusion
    start = tr.perturb(tr.aa_to_rt(c2["poses_true"])[TRACK_IDS], 0.5, 0.005, seed=13)
    # one schedule: planes on every level, the first system at level 2, the last at level 0
    with _Clock() as cr:
        out, frames = _check_rgbd_against_restatement(e, c2, TRACK_IDS, start, 3, (3, 2, 1), PHOTO)
    rows = [(i["color"]["first_rows"], i["color"]["last_rows"]) for i in out[1]]
    tiles = _tiles(e.debug_track_color_planes(0, len(TRACK_IDS), model_intensity=False)["intensity"])
    assert tiles == 1200 and all(last > 10_000 for _, last in rows), rows
    _report(13, schedule=(3, 2, 1), tiles_level0=tiles, photometric_rows=rows, correspondences=[i["correspondences"] for i in out[1]],
            device_ms=e.phase_ms("track"), cpu_s_with_engine_call=cr.s)
