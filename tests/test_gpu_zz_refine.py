"""nv::Intrinsic3D::refine (reference-shaped orchestrator on ONE resident engine):
  (1) against the float64 ORACLE driven through the same two-level schedule (src/refinement/intrinsic3d.cpp:206-295: convert -> initial
      recolouring -> per grid level {thin-shell pruning -> per pyramid level {lighting, GN iterations, recolouring} -> upsample}),
  (2) against the same schedule driven from Python through the C-ABI (same engine: isolates the C++ host code).
A voxel on the pruning threshold can flip between two runs (float atomics in the engine, f32 Jacobian vs the oracle's f64), so the
comparison is on counts (within 0.5 %) and, for the voxels both runs hold, on the distribution of the differences."""
import ctypes as C
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GL, RL, ITS = 2, 2, 2
FACTOR0, FACTOR1 = 2.0, 1.0
LAM = dict(g=0.2, r0=80.0, r1=10.0, s0=120.0, s1=10.0, a=0.1)
SUB_SIZE, SH_REG, OCCL, K = 0.06, 10.0, 0.02, 5


def _lam(it, n, a, b):
    return a if n <= 1 else a + (b - a) * it / (n - 1)          # computeVaryingLambda (include/nv/refinement/cost.h)


def _setup():
    from intrinsic3d_b200.scene import make_color_frames, make_scene
    s = make_scene(radius_vox=12.0, frames=6, width=160, height=120, voxel_size=0.008, band=3.0, seed=6)
    col = make_color_frames(s)
    F, H, W = s["lum"].shape
    lum1 = s["lum"].reshape(F, H // 2, 2, W // 2, 2).mean((2, 4)).astype(np.float32)
    dep1 = np.ascontiguousarray(s["depth"][:, ::2, ::2])
    return s, col, lum1, dep1


class _EngineDriver:
    def __init__(self, s, col):
        from intrinsic3d_b200 import engine
        keep = s["weight"] > 0
        self.e = e = engine.Engine(0)
        sdf = s["sdf0"][keep].astype(np.float32).astype(np.float64)
        e.upload_grid(s["xyz"][keep], sdf, sdf, np.full(int(keep.sum()), 0.6), s["weight"][keep], s["rgb"][keep], s["voxel_size"])
        e.upload_frames(s["lum"], s["depth"], 1.0)
        e.upload_color_frames(col)
        e.set_camera(s["poses"], np.ascontiguousarray(s["intr"], np.float64), np.zeros(5))
        self.LP = engine.default_lighting_params()
        self.col = col

    def frames(self, lum, depth, scale, level0):
        self.e.upload_frames(lum, depth, scale)
        if level0:
            self.e.upload_color_frames(self.col)

    def grid(self):
        return self.e.download_grid()

    def state(self):
        return self.e.download_state()

    def __getattr__(self, k):
        return getattr(self.e, k)


class _OracleDriver:
    def __init__(self, s, col):
        import oracle
        keep = s["weight"] > 0
        n = int(keep.sum())
        sdf = s["sdf0"][keep].astype(np.float32).astype(np.float64)
        so = dict(xyz=s["xyz"][keep], sdf0=sdf, sdf_refined=sdf.copy(), albedo=np.full(n, 0.6), weight=s["weight"][keep], rgb=s["rgb"][keep],
                  voxel_size=s["voxel_size"], lum=s["lum"], depth=s["depth"], poses=s["poses"], intr=np.ascontiguousarray(s["intr"], np.float64),
                  dist=np.zeros(5), sh=np.zeros((n, 9)))
        self.o = o = oracle.Oracle(threads=8)
        o.load_scene(so)
        o.set_color_frames(col)
        self.LP = oracle.default_lighting_params()
        self.col = col

    def frames(self, lum, depth, scale, level0):
        self.o.set_frames(lum, depth, scale)
        if level0:
            self.o.set_color_frames(self.col)

    def grid(self):
        return self.o.grid()

    def __getattr__(self, k):
        return getattr(self.o, k)


def _schedule(d, s, lum1, dep1):
    """Intrinsic3D::refine's control flow on a driver (engine through the C-ABI, or the oracle)."""
    from intrinsic3d_b200.ctypes_defs import default_params
    d.recompute_colors(OCCL, K)
    vs = float(np.float32(s["voxel_size"]))
    LP = d.LP
    LP.subvolume_size = SUB_SIZE; LP.lambda_reg = SH_REG; LP.weighted = 1
    level = 0
    for gl in range(GL - 1, -1, -1):
        fac = _lam(GL - 1 - gl, GL, FACTOR0, FACTOR1)
        thres = fac * vs
        d.clear_voxels_outside_thin_shell(thres)
        for rl in range(RL - 1, -1, -1):
            if rl > 0 and gl < GL - 1:
                continue
            if rl != level:
                d.frames(lum1 if rl == 1 else s["lum"], dep1 if rl == 1 else s["depth"], 1.0 / 2 ** rl, rl == 0)
                level = rl
            LP.thres_shell = thres
            li = d.estimate_lighting(LP)
            assert li.usable == 1
            for it in range(ITS):
                p = default_params()
                p.thres_shell = thres; p.occlusion_distance = OCCL; p.num_observations = K
                p.lambda_[0] = LAM["g"]; p.lambda_[1] = _lam(it, ITS, LAM["r0"], LAM["r1"]); p.lambda_[2] = _lam(it, ITS, LAM["s0"], LAM["s1"]); p.lambda_[3] = LAM["a"]
                d.gn_iteration(p)
            if level != 0:
                d.frames(s["lum"], s["depth"], 1.0, True); level = 0
            d.recompute_colors(OCCL, K)
        if gl > 0:
            d.upsample_grid()
            vs = float(np.float32(np.float32(vs) * np.float32(0.5)))
    return d.grid(), d.state()


def _run_cpp(s, col, lum1, dep1):
    Hh = C.CDLL(os.path.join(ROOT, "intrinsic3d_b200", "libi3d_host.so"))

    def ptr(a, t):
        return a.ctypes.data_as(C.POINTER(t))
    F, H, W = s["lum"].shape
    n = len(s["xyz"])
    xyz = np.ascontiguousarray(s["xyz"], np.int32)
    sdf = np.ascontiguousarray(s["sdf0"], np.float32)
    wgt = np.ascontiguousarray(s["weight"], np.float32)
    rgb = np.ascontiguousarray(s["rgb"], np.uint8)
    lum0 = np.ascontiguousarray(s["lum"], np.float32); dep0 = np.ascontiguousarray(s["depth"], np.float32)
    Wl = np.array([W, W // 2], np.int32); Hl = np.array([H, H // 2], np.int32)
    lum_ptrs = (C.POINTER(C.c_float) * 2)(ptr(lum0, C.c_float), ptr(lum1, C.c_float))
    dep_ptrs = (C.POINTER(C.c_float) * 2)(ptr(dep0, C.c_float), ptr(dep1, C.c_float))
    colc = np.ascontiguousarray(col, np.uint8)
    poses = np.ascontiguousarray(s["poses"], np.float64).copy()
    intr = np.ascontiguousarray(s["intr"], np.float64).copy(); dist = np.zeros(5)
    cfg = np.array([GL, RL, FACTOR0, FACTOR1, 1, OCCL, K, SUB_SIZE, SH_REG, ITS, 50, LAM["g"], LAM["r0"], LAM["r1"], LAM["s0"], LAM["s1"], LAM["a"]], np.float64)
    cap = 8 * n
    out = dict(xyz=np.zeros((cap, 3), np.int32), sdf0=np.zeros(cap), sdf=np.zeros(cap), alb=np.zeros(cap), w=np.zeros(cap, np.float32), rgb=np.zeros((cap, 3), np.uint8))
    m = C.c_int64(0); vso = C.c_float(0); calls = C.c_int32(0)
    rc = Hh.i3dh_run_refine(C.c_int64(n), ptr(xyz, C.c_int32), ptr(sdf, C.c_float), ptr(wgt, C.c_float), ptr(rgb, C.c_uint8), C.c_float(float(s["voxel_size"])),
                            C.c_int32(F), C.c_int32(2), ptr(Wl, C.c_int32), ptr(Hl, C.c_int32), lum_ptrs, dep_ptrs, ptr(colc, C.c_uint8), ptr(poses, C.c_double),
                            ptr(intr, C.c_double), ptr(dist, C.c_double), ptr(cfg, C.c_double), C.c_int64(cap), C.byref(m), ptr(out["xyz"], C.c_int32),
                            ptr(out["sdf0"], C.c_double), ptr(out["sdf"], C.c_double), ptr(out["alb"], C.c_double), ptr(out["w"], C.c_float), ptr(out["rgb"], C.c_uint8),
                            C.byref(vso), C.byref(calls))
    assert rc == 0
    M = int(m.value)
    assert calls.value == 3                                # (gl 1: rl 1, rl 0) + (gl 0: rl 0)
    res = dict(xyz=out["xyz"][:M], sdf0=out["sdf0"][:M], sdf_refined=out["sdf"][:M], albedo=out["alb"][:M], weight=out["w"][:M], rgb=out["rgb"][:M], voxel_size=np.float32(vso.value))
    return res, dict(poses=poses, intr=intr, dist=dist)


def _compare(ref, ref_state, out, out_state, s):
    """distribution of the differences over the voxels both results hold, relative to the size of the refinement itself"""
    M = len(out["xyz"])
    a = {tuple(c): i for i, c in enumerate(ref["xyz"])}
    common = [(a[tuple(c)], i) for i, c in enumerate(out["xyz"]) if tuple(c) in a]
    ia, ib = np.array(common).T
    moved = float(np.abs(ref["sdf_refined"] - ref["sdf0"]).max())
    d = np.abs(ref["sdf_refined"][ia] - out["sdf_refined"][ib]) / moved
    da = np.abs(ref["albedo"][ia] - out["albedo"][ib])
    dc = np.abs(ref["rgb"][ia].astype(int) - out["rgb"][ib].astype(int)).max(1)
    return dict(voxels_ref=int(len(ref["xyz"])), voxels_out=M, common=int(len(common)), sdf_update_max=moved,
                sdf_err_rel_median=float(np.median(d)), sdf_err_rel_p98=float(np.quantile(d, 0.98)), sdf_err_rel_max=float(d.max()),
                sdf_frac_within_1e3=float((d <= 1e-3).mean()), sdf_frac_within_1e2=float((d <= 1e-2).mean()),
                albedo_err_median=float(np.median(da)), albedo_err_p98=float(np.quantile(da, 0.98)), albedo_frac_within_1e3=float((da <= 1e-3).mean()),
                color_frac_within_1=float((dc <= 1).mean()),
                pose_err_max=float(np.abs(out_state["poses"] - ref_state["poses"]).max()), pose_update_max=float(np.abs(ref_state["poses"] - s["poses"]).max()),
                intr_err_max=float(np.abs(out_state["intr"] - ref_state["intr"]).max()), intr_update_max=float(np.abs(ref_state["intr"] - s["intr"]).max()))


def test_cpp_refine_matches_oracle_schedule():
    """(1) the C++ orchestrator on the engine vs the float64 oracle driven through the same schedule: 6 GN iterations over 2 grid levels /
    2 pyramid levels with lighting, recolouring, pruning and upsampling in between — including the camera state across the level switches."""
    s, col, lum1, dep1 = _setup()
    ref, ref_state = _schedule(_OracleDriver(s, col), s, lum1, dep1)
    out, out_state = _run_cpp(s, col, lum1, dep1)
    assert out["voxel_size"] == ref["voxel_size"] == np.float32(np.float32(s["voxel_size"]) * np.float32(0.5))
    r = _compare(ref, ref_state, out, out_state, s)
    print("test_refine_vs_oracle:", json.dumps(r))
    assert abs(r["voxels_out"] - r["voxels_ref"]) <= 0.005 * r["voxels_ref"] and r["common"] >= 0.995 * r["voxels_out"]
    # the bounds leave a margin for float-atomic run-to-run differences
    assert r["sdf_update_max"] > 0 and r["sdf_err_rel_median"] <= 1e-4 and r["sdf_frac_within_1e3"] > 0.99 and r["sdf_frac_within_1e2"] > 0.999
    assert r["albedo_frac_within_1e3"] > 0.99 and r["color_frac_within_1"] > 0.99
    assert r["pose_update_max"] > 1e-4 and r["pose_err_max"] <= 1e-3 * r["pose_update_max"]
    assert r["intr_err_max"] <= 1e-3 * max(r["intr_update_max"], 1e-3)


def test_cpp_refine_matches_python_driven_schedule():
    """(2) the C++ host code in isolation: same engine, schedule driven from Python through the C-ABI."""
    s, col, lum1, dep1 = _setup()
    ref, ref_state = _schedule(_EngineDriver(s, col), s, lum1, dep1)
    out, out_state = _run_cpp(s, col, lum1, dep1)
    n = len(s["xyz"])
    M = len(out["xyz"])
    assert out["voxel_size"] == ref["voxel_size"] == np.float32(np.float32(s["voxel_size"]) * np.float32(0.5))
    assert abs(M - len(ref["xyz"])) <= 0.005 * len(ref["xyz"]) and M > 8 * 0.1 * n
    r = _compare(ref, ref_state, out, out_state, s)
    assert r["common"] >= 0.995 * M
    assert r["sdf_update_max"] > 0 and r["sdf_frac_within_1e3"] > 0.98, r
    assert r["albedo_frac_within_1e3"] > 0.98
    assert r["color_frac_within_1"] > 0.97
    assert r["pose_err_max"] < 1e-4 and r["intr_err_max"] < 1e-2
    assert not np.allclose(out_state["poses"], s["poses"])
