"""The normal-equation kernels entry by entry against a float64 reference of the same operation (tests/normal_equations_ref.py):
gradient b = J'^T f, Jacobi scale s, jtj = s^2 colnorm^2, the raw camera sums cam_acc that k_cam_precond inverts, and single
applications of the CGNR operator q = S J^T W J S v (k_eg_apply + k_op_partial), at the shapes where these kernels go wrong.

The reference is built from the engine's own E_g rows (float32 J, raw weights, frames) and the oracle's regulariser rows (pinned
equal to the engine's by test_gpu_parity.py), so the bound |gpu - ref|_j <= c 2^-24 M_j (M_j: the same sums over absolute values,
c: float roundings of the kernel's chain, normal_equations_ref.rounding_counts) measures nothing but the kernels' arithmetic.
"""
import json
import os
import re

import numpy as np
import pytest

import normal_equations_ref as ner

pytestmark = pytest.mark.gpu


def _params(scene, **kw):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = scene["thres_shell"]
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _note(name, payload):
    """the achieved max(err / bound) per quantity, in the test's captured output (pytest -rA shows them)"""
    print(f"test_{name}:", json.dumps(payload))


def _vectors(R, rows, seed=11):
    """a seeded random vector and unit vectors on a pose column (the most observed frame), an intrinsics and a distortion column"""
    rng = np.random.default_rng(seed)
    vs = [rng.standard_normal(R.U).astype(np.float32)]
    f = int(np.bincount(rows["frame"]).argmax()) if len(rows["frame"]) else 0
    for j in (2 * R.n + 6 * f + 3, 2 * R.n + 6 * R.F + 1, 2 * R.n + 6 * R.F + 4):
        e = np.zeros(R.U, np.float32)
        e[j] = 1.0
        vs.append(e)
    return vs


def check_normal_equations(scene, p, name, e=None):
    """One build-only iteration of engine and oracle on `scene`; every quantity compared against the reference.  Returns the
    per-quantity max(err / bound)."""
    from intrinsic3d_b200.engine import Engine
    from oracle import Oracle
    if e is None:
        e = Engine(0)
        e.load_scene(scene)
    p = type(p).from_buffer_copy(bytes(p))
    p.build_only = 1
    ie = e.gn_iteration(p)
    o = Oracle(threads=min(32, os.cpu_count() or 8))
    o.load_scene(scene)
    io = o.gn_iteration(p)
    assert list(ie.type_residuals) == list(io.type_residuals) and ie.num_active == io.num_active
    K = p.num_observations if 0 < p.num_observations <= scene["poses"].shape[0] else scene["poses"].shape[0]
    rows = e.debug_rows()
    stride = len(rows["frame"]) // max(K, 1)
    ok = rows["frame"] >= 0
    sl = np.nonzero(ok)[0]
    tw = np.array(list(ie.type_weights))
    eg = dict(voxel=rows["voxel"][sl], frame=rows["frame"][sl], residual=rows["residual"][sl], raw_weight=rows["raw_weight"][sl],
              J=rows["J"][:, sl].T.astype(np.float64), slot=sl % stride,
              w_op=np.float32(rows["raw_weight"][sl] * tw[0]).astype(np.float64))      # k_row_weights
    # same E_g row set as the oracle's
    ro = o.rows(0)
    assert set(zip(eg["voxel"].tolist(), eg["frame"].tolist())) == set(zip(ro["voxel"].tolist(), ro["aux"].tolist()))
    R = ner.build_rows(scene, eg, (o.rows(1), o.rows(2), o.rows(3)), tw)
    free = o.step()[1].astype(bool)
    ne = e.debug_normal_equations()
    vs = _vectors(R, eg)
    qs = [e.debug_apply_operator(v) for v in vs]
    ref = ner.evaluate(R, free, ne["s"], vs)
    c = ner.rounding_counts(K)
    got = dict(s=ne["s"], jtj=ne["jtj"], b=ne["b"], cam_acc=ne["cam_acc"])
    got.update({f"q{i}": q for i, q in enumerate(qs)})
    res, bad = {}, {}
    for k, x in got.items():
        ratio, good, nbad = ner.compare(x, ref[k], c["q" if k.startswith("q") else k])
        res[k] = ratio
        if not good:
            bad[k] = nbad
    # structural zeros beyond the bound: fixed unknowns and frames no row sees
    assert np.all(ne["s"][~free] == 0) and np.all(ne["b"][~free] == 0) and all(np.all(q[~free] == 0) for q in qs)
    seen = np.bincount(eg["frame"], minlength=R.F) > 0
    assert np.all(ne["cam_acc"][:33 * R.F].reshape(R.F, 33)[~seen] == 0)
    _note(f"normal_equations[{name}]", dict(K=K, n_active=int(ie.num_active), frames=R.F, eg_rows=int(len(sl)),
                                             frames_seen=int(seen.sum()), max_err_over_bound=res))
    assert not bad, (name, bad, res)
    return res


def _active_cut(scene, target, base_params):
    """thres_shell that leaves exactly `target` active voxels (the count grows by at most one voxel per |sdf| value)"""
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(scene)
    vals = np.unique(np.abs(scene["sdf_refined"]))
    p = type(base_params).from_buffer_copy(bytes(base_params))
    p.build_only = 1

    def count(i):
        p.thres_shell = float(vals[i])
        return int(e.gn_iteration(p).num_active)

    lo, hi = 0, len(vals) - 1
    while lo < hi:
        mid = (lo + hi) // 2
        if count(mid) < target:
            lo = mid + 1
        else:
            hi = mid
    assert count(lo) == target
    return float(vals[lo])


@pytest.mark.parametrize("K", [1, 5, 8])
def test_observations_per_voxel(K, small_scene):
    """k_select_obs<5> vs <8>; K = 8 takes the > 48 KB dynamic shared-memory path of k_eg_accum and k_eg_apply"""
    check_normal_equations(small_scene, _params(small_scene, num_observations=K), f"K{K}")


@pytest.mark.parametrize("n_active", [1, 31, 33, 257])
def test_few_active_voxels(n_active, tiny_scene):
    """partial warps: the distinct-frame walk and the reduce-scatter with idle lanes, the stride padding"""
    p = _params(tiny_scene)
    p.thres_shell = _active_cut(tiny_scene, n_active, p)
    s = dict(tiny_scene)
    s["thres_shell"] = p.thres_shell
    check_normal_equations(s, p, f"n_active{n_active}")


def test_many_frames_per_warp():
    """64 small frames around the object, K = 8: many distinct frames in one warp's rows"""
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("tiny", frames=64, width=64, height=48)
    check_normal_equations(s, _params(s, num_observations=8), "64_frames_K8")


SWITCHES = [dict(fix_poses=1), dict(fix_intrinsics=1), dict(fix_distortion=1), dict(fix_all_albedo=1),
            dict(use_er=0), dict(use_es=0), dict(use_ea=0)]


@pytest.mark.parametrize("sw", SWITCHES, ids=lambda d: "_".join(f"{k}{v}" for k, v in d.items()))
def test_switches(sw, tiny_scene):
    s = dict(tiny_scene)
    s["dist"] = np.array([0.02, -0.01, 0.003, 0.001, -0.0007])
    check_normal_equations(s, _params(s, **sw), "_".join(f"{k}{v}" for k, v in sw.items()))


def test_invalid_and_black_voxels(tiny_scene):
    """the scene of test_edge_cases_match_oracle: weight-0 voxels, black voxels (NaN albedo-pair weights), a coarser pyramid level"""
    s = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in tiny_scene.items()}
    rng = np.random.default_rng(7)
    n = s["xyz"].shape[0]
    s["weight"][rng.choice(n, n // 50, replace=False)] = 0.0
    s["rgb"][rng.choice(n, n // 40, replace=False)] = 0
    s["dist"] = np.array([0.02, -0.01, 0.003, 0.001, -0.0007])
    s["intr"] = s["intr"] * 2.0
    s["pyr_scale"] = 0.5
    check_normal_equations(s, _params(s, num_observations=8), "invalid_black")


def test_c3_slab_many_blocks():
    """the C3 1/16 z-slab with all 200 frames: thousands of blocks add camera partials into the same entries"""
    import torch
    from bench import slab_scene
    from intrinsic3d_b200.scene import config_scene
    s, _ = slab_scene(config_scene("c3", device="cuda" if torch.cuda.is_available() else "cpu"), 1.0 / 16.0)
    check_normal_equations(s, _params(s), "c3_slab")


def _max_frames(scene, K):
    """the largest frame count i3d_gn_iteration accepts at K, from its error message on 1000 blank frames"""
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(scene)
    F = 1000
    e.upload_frames(np.zeros((F, 24, 32), np.float32), np.zeros((F, 24, 32), np.float32))
    e.set_camera(np.zeros((F, 6)), scene["intr"], scene["dist"])
    with pytest.raises(RuntimeError) as ex:
        e.gn_iteration(_params(scene, num_observations=K, build_only=1))
    msg = str(ex.value)
    assert f"{F} frames at K = {K}" in msg, msg
    return int(re.search(r"at most (\d+) frames", msg).group(1))


def test_frame_count_at_shared_memory_limit(tiny_scene):
    """the largest accepted F at K = 8 passes the comparison; F + 1 is refused with a message naming F, K and the limit, and the
    engine stays usable"""
    from intrinsic3d_b200.engine import Engine
    from intrinsic3d_b200.scene import config_scene
    K = 8
    fmax = _max_frames(tiny_scene, K)
    assert 500 <= fmax < 1000
    s = config_scene("tiny", frames=fmax, width=32, height=24)
    e = Engine(0)
    e.load_scene(s)
    check_normal_equations(s, _params(s, num_observations=K), f"F{fmax}_K{K}", e=e)
    lum = np.concatenate([s["lum"], s["lum"][:1]])
    depth = np.concatenate([s["depth"], s["depth"][:1]])
    poses = np.concatenate([s["poses"], s["poses"][:1]])
    e.upload_frames(lum, depth)
    e.set_camera(poses, s["intr"], s["dist"])
    with pytest.raises(RuntimeError) as ex:
        e.gn_iteration(_params(s, num_observations=K))
    msg = str(ex.value)
    assert f"{fmax + 1} frames at K = {K}" in msg and f"at most {fmax} frames" in msg, msg
    # still usable: the same frames at K = 5, then back to fmax frames at K = 8
    info = e.gn_iteration(_params(s, num_observations=5, forced_cg_iterations=2))
    assert info.num_active > 0 and info.lm_iterations >= 1
    e.upload_frames(s["lum"], s["depth"])
    e.set_camera(s["poses"], s["intr"], s["dist"])
    info = e.gn_iteration(_params(s, num_observations=K, forced_cg_iterations=2))
    assert info.lm_iterations >= 1


def test_operator_leaves_no_state_behind(small_scene):
    """an operator application between two iterations changes nothing the following iteration computes"""
    from intrinsic3d_b200.engine import Engine
    s = small_scene
    outs = []
    for with_operator in (False, True):
        e = Engine(0)
        e.load_scene(s)
        p = _params(s)
        e.gn_iteration(p)
        if with_operator:
            U = 2 * e.n + 6 * e.F + 9
            e.debug_apply_operator(np.random.default_rng(5).standard_normal(U).astype(np.float32))
        info = e.gn_iteration(p)
        st = e.download_state()
        outs.append((st, info, e.debug_normal_equations(), e.debug_step()))
        e.close()
    (a, ia, na, da), (b, ib, nb, db) = outs
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    for k in na:
        assert na[k].tobytes() == nb[k].tobytes(), k
    for x, y in zip(da, db):
        assert x.tobytes() == y.tobytes()
    assert iter_info_bytes(ia) == iter_info_bytes(ib)


def iter_info_bytes(info):
    """the bytes of every I3DIterInfo field before the wall-clock timers (time_add, time_build, time_solve come last)"""
    return bytes(info)[:type(info).time_add.offset]
