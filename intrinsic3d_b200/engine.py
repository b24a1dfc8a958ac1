"""Python host-side binding of the C-ABI in include/i3d_c_api.h (libi3d_b200.so).

This is plumbing for tests and bench.py: it passes HOST numpy buffers through the same
extern "C" entry points a C++ caller (include/nv/refinement/ shims) uses.  There is no CPU
fallback: if the CUDA library is missing or no sm_90 (H100) device is present, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .ctypes_defs import I3DIterInfo, I3DLightingInfo, I3DLightingParams, I3DParams

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("I3D_LIB", os.path.join(_HERE, "libi3d_b200.so"))   # I3D_LIB: A/B builds of the same library
_LIB = None

EXPORTED_SYMBOLS = [
    "i3d_abi_version", "i3d_sizeof_params", "i3d_sizeof_iter_info", "i3d_default_params",
    "i3d_engine_create", "i3d_engine_destroy", "i3d_last_error",
    "i3d_upload_grid", "i3d_upload_voxel_params", "i3d_upload_frames", "i3d_set_camera", "i3d_set_sh",
    "i3d_gn_iteration", "i3d_download_state",
    "i3d_sizeof_lighting_params", "i3d_sizeof_lighting_info", "i3d_default_lighting_params", "i3d_estimate_lighting",
    "i3d_lighting_num_subvolumes", "i3d_download_lighting", "i3d_download_voxel_sh",
    "i3d_upload_color_frames", "i3d_recompute_colors", "i3d_download_colors",
    "i3d_num_voxels", "i3d_clear_voxels_outside_thin_shell", "i3d_upsample_grid", "i3d_download_grid",
    "i3d_comm_unique_id", "i3d_comm_init", "i3d_comm_p2p_export", "i3d_comm_p2p_connect", "i3d_set_shard",
    "i3d_phase_ms", "i3d_phase_count", "i3d_debug_set_kernel_timers", "i3d_debug_num_slots", "i3d_debug_set_keep_raw_jacobian",
    "i3d_debug_get_rows", "i3d_debug_get_observations", "i3d_debug_get_step", "i3d_debug_get_normal_equations",
    "i3d_debug_apply_operator",
]


def load_library():
    """Loads libi3d_b200.so.  Raises (never falls back) when the CUDA extension is missing."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: build it with intrinsic3d_b200/csrc/build.sh "
                           "(__graft_entry__.build()); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    L.i3d_abi_version.restype = C.c_int
    L.i3d_sizeof_params.restype = C.c_uint64
    L.i3d_sizeof_iter_info.restype = C.c_uint64
    L.i3d_last_error.restype = C.c_char_p
    L.i3d_last_error.argtypes = [C.c_void_p]
    L.i3d_phase_ms.restype = C.c_double
    L.i3d_phase_ms.argtypes = [C.c_void_p, C.c_char_p]
    L.i3d_phase_count.restype = C.c_int64
    L.i3d_phase_count.argtypes = [C.c_void_p, C.c_char_p]
    L.i3d_debug_num_slots.restype = C.c_int64
    L.i3d_debug_num_slots.argtypes = [C.c_void_p]
    L.i3d_sizeof_lighting_params.restype = C.c_uint64
    L.i3d_sizeof_lighting_info.restype = C.c_uint64
    L.i3d_lighting_num_subvolumes.restype = C.c_int64
    L.i3d_lighting_num_subvolumes.argtypes = [C.c_void_p]
    L.i3d_num_voxels.restype = C.c_int64
    L.i3d_num_voxels.argtypes = [C.c_void_p]
    if L.i3d_sizeof_params() != C.sizeof(I3DParams) or L.i3d_sizeof_iter_info() != C.sizeof(I3DIterInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so")
    if L.i3d_sizeof_lighting_params() != C.sizeof(I3DLightingParams) or L.i3d_sizeof_lighting_info() != C.sizeof(I3DLightingInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (lighting structs)")
    _LIB = L
    return L


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def default_params() -> I3DParams:
    p = I3DParams()
    load_library().i3d_default_params(C.byref(p))
    return p


def default_lighting_params() -> I3DLightingParams:
    p = I3DLightingParams()
    load_library().i3d_default_lighting_params(C.byref(p))
    return p


class Engine:
    """One GPU-resident problem: grid + frames + camera + SH; gn_iteration() = one outer GN iteration."""

    def __init__(self, device: int = 0):
        self.L = load_library()
        h = C.c_void_p()
        rc = self.L.i3d_engine_create(C.c_int(device), C.byref(h))
        if rc != 0:
            raise RuntimeError("i3d_engine_create failed: " + self.L.i3d_last_error(None).decode())
        self.h = h
        self.n = 0
        self.F = 0

    def close(self):
        if getattr(self, "h", None):
            self.L.i3d_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.i3d_last_error(self.h).decode())

    # ---- uploads (host buffers; copied during the call) -------------------------------------
    def upload_grid(self, xyz, sdf0, sdf_refined, albedo, weight, rgb, voxel_size):
        xyz = np.ascontiguousarray(xyz, np.int32)
        n = int(xyz.shape[0])
        a = [np.ascontiguousarray(sdf0, np.float64), np.ascontiguousarray(sdf_refined, np.float64),
             np.ascontiguousarray(albedo, np.float64), np.ascontiguousarray(weight, np.float32),
             np.ascontiguousarray(rgb, np.uint8)]
        self._check(self.L.i3d_upload_grid(self.h, C.c_int64(n), _p(xyz, C.c_int32), _p(a[0], C.c_double), _p(a[1], C.c_double),
                                           _p(a[2], C.c_double), _p(a[3], C.c_float), _p(a[4], C.c_uint8), C.c_float(float(voxel_size))))
        self.n = n

    def upload_voxel_params(self, sdf_refined, albedo):
        s = np.ascontiguousarray(sdf_refined, np.float64)
        a = np.ascontiguousarray(albedo, np.float64)
        self._check(self.L.i3d_upload_voxel_params(self.h, _p(s, C.c_double), _p(a, C.c_double)))

    def upload_frames(self, lum, depth, pyr_scale=1.0):
        lum = np.ascontiguousarray(lum, np.float32)
        depth = np.ascontiguousarray(depth, np.float32)
        F, H, W = lum.shape
        self._check(self.L.i3d_upload_frames(self.h, C.c_int32(F), C.c_int32(W), C.c_int32(H), _p(lum, C.c_float), _p(depth, C.c_float),
                                             C.c_double(float(pyr_scale))))
        self.F = F

    def set_camera(self, poses, intr, dist):
        poses = np.ascontiguousarray(poses, np.float64)
        intr = np.ascontiguousarray(intr, np.float64)
        dist = np.ascontiguousarray(dist, np.float64)
        self._check(self.L.i3d_set_camera(self.h, _p(poses, C.c_double), _p(intr, C.c_double), _p(dist, C.c_double)))

    def set_sh(self, sh):
        sh = np.ascontiguousarray(sh, np.float64)
        assert sh.shape == (self.n, 9)
        self._check(self.L.i3d_set_sh(self.h, _p(sh, C.c_double)))

    def load_scene(self, s):
        self.upload_grid(s["xyz"], s["sdf0"], s["sdf_refined"], s["albedo"], s["weight"], s["rgb"], s["voxel_size"])
        self.upload_frames(s["lum"], s["depth"], s.get("pyr_scale", 1.0))
        self.set_camera(s["poses"], s["intr"], s["dist"])
        self.set_sh(s["sh"])

    # ---- compute ----------------------------------------------------------------------------
    def gn_iteration(self, params: I3DParams) -> I3DIterInfo:
        info = I3DIterInfo()
        self._check(self.L.i3d_gn_iteration(self.h, C.byref(params), C.byref(info)))
        return info

    # ---- SVSH lighting (LightingSVSH::estimate + computeVoxelShCoeffs) -----------------------
    def estimate_lighting(self, params: I3DLightingParams) -> I3DLightingInfo:
        """Estimates the subvolume SH on the uploaded grid and leaves the per-voxel blend as the engine's `sh` input."""
        info = I3DLightingInfo()
        self._check(self.L.i3d_estimate_lighting(self.h, C.byref(params), C.byref(info)))
        return info

    def download_lighting(self):
        S = int(self.L.i3d_lighting_num_subvolumes(self.h))
        idx = np.empty((S, 3), np.int32)
        sh = np.empty((S, 9), np.float64)
        self._check(self.L.i3d_download_lighting(self.h, _p(idx, C.c_int32), _p(sh, C.c_double)))
        return idx, sh

    def download_voxel_sh(self):
        sh = np.empty((self.n, 9), np.float64)
        has = np.empty(self.n, np.uint8)
        self._check(self.L.i3d_download_voxel_sh(self.h, _p(sh, C.c_double), _p(has, C.c_uint8)))
        return sh, has

    # ---- voxel recolouring (Intrinsic3D::recomputeColors) ------------------------------------
    def upload_color_frames(self, bgr):
        bgr = np.ascontiguousarray(bgr, np.uint8)
        assert bgr.ndim == 4 and bgr.shape[0] == self.F and bgr.shape[3] == 3
        self._check(self.L.i3d_upload_color_frames(self.h, _p(bgr, C.c_uint8)))

    def recompute_colors(self, max_occlusion_distance: float = 0.02, max_num_observations: int = 5, pose_rt=None):
        """Returns (voxels recoloured, observations with weight > 0).  pose_rt: optional float32 [F, 12] (R row-major | t)."""
        a, b = C.c_int64(0), C.c_int64(0)
        if pose_rt is not None:
            pose_rt = np.ascontiguousarray(pose_rt, np.float32)
            assert pose_rt.shape == (self.F, 12)
        self._check(self.L.i3d_recompute_colors(self.h, _p(pose_rt, C.c_float), C.c_float(max_occlusion_distance), C.c_int32(max_num_observations),
                                                C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def download_colors(self):
        rgb = np.empty((self.n, 3), np.uint8)
        self._check(self.L.i3d_download_colors(self.h, _p(rgb, C.c_uint8)))
        return rgb

    # ---- grid-level transitions (SDFAlgorithms::clearVoxelsOutsideThinShell / upsample) -------
    def clear_voxels_outside_thin_shell(self, thres_shell: float) -> int:
        m = C.c_int64(0)
        self._check(self.L.i3d_clear_voxels_outside_thin_shell(self.h, C.c_double(thres_shell), C.byref(m)))
        self.n = int(m.value)
        return self.n

    def upsample_grid(self) -> int:
        m = C.c_int64(0)
        self._check(self.L.i3d_upsample_grid(self.h, C.byref(m)))
        self.n = int(m.value)
        return self.n

    def download_grid(self):
        n = int(self.L.i3d_num_voxels(self.h))
        out = dict(xyz=np.empty((n, 3), np.int32), sdf0=np.empty(n, np.float64), sdf_refined=np.empty(n, np.float64), albedo=np.empty(n, np.float64),
                   weight=np.empty(n, np.float32), rgb=np.empty((n, 3), np.uint8))
        vs = C.c_float(0)
        self._check(self.L.i3d_download_grid(self.h, _p(out["xyz"], C.c_int32), _p(out["sdf0"], C.c_double), _p(out["sdf_refined"], C.c_double),
                                             _p(out["albedo"], C.c_double), _p(out["weight"], C.c_float), _p(out["rgb"], C.c_uint8), C.byref(vs)))
        out["voxel_size"] = np.float32(vs.value)
        return out

    def download_state(self):
        sdf = np.empty(self.n, np.float64)
        alb = np.empty(self.n, np.float64)
        poses = np.empty((self.F, 6), np.float64)
        intr = np.empty(4, np.float64)
        dist = np.empty(5, np.float64)
        self._check(self.L.i3d_download_state(self.h, _p(sdf, C.c_double), _p(alb, C.c_double), _p(poses, C.c_double),
                                              _p(intr, C.c_double), _p(dist, C.c_double)))
        return dict(sdf_refined=sdf, albedo=alb, poses=poses, intr=intr, dist=dist)

    # ---- measurement / parity hooks ---------------------------------------------------------
    def phase_ms(self, name: str) -> float:
        return float(self.L.i3d_phase_ms(self.h, name.encode()))

    def phase_count(self, name: str) -> int:
        return int(self.L.i3d_phase_count(self.h, name.encode()))

    def set_kernel_timers(self, level: int):
        """0 (default): phases + the roofline kernels (first k_eg_apply of each solve); 1: every kernel of the iteration."""
        self.L.i3d_debug_set_kernel_timers(self.h, C.c_int(int(level)))

    def debug_rows(self, want_jac=True):
        S = int(self.L.i3d_debug_num_slots(self.h))
        voxel = np.empty(S, np.int32)
        frame = np.empty(S, np.int32)
        res = np.empty(S, np.float64)
        w = np.empty(S, np.float64)
        J = np.empty((29, S), np.float32) if want_jac else None
        self._check(self.L.i3d_debug_get_rows(self.h, _p(voxel, C.c_int32), _p(frame, C.c_int32), _p(res, C.c_double), _p(w, C.c_double),
                                              _p(J, C.c_float)))
        return dict(voxel=voxel, frame=frame, residual=res, raw_weight=w, J=J)

    def debug_observations(self, K: int):
        fr = np.empty((self.n, K), np.int32)
        w = np.empty((self.n, K), np.float32)
        act = np.empty(self.n, np.uint8)
        self._check(self.L.i3d_debug_get_observations(self.h, C.c_int32(K), _p(fr, C.c_int32), _p(w, C.c_float), _p(act, C.c_uint8)))
        return fr, w, act

    def debug_step(self):
        U = 2 * self.n + 6 * self.F + 9
        st = np.zeros(U, np.float64)
        fm = np.zeros(U, np.uint8)
        cs = np.zeros(U, np.float64)
        self._check(self.L.i3d_debug_get_step(self.h, _p(st, C.c_double), _p(fm, C.c_uint8), _p(cs, C.c_double)))
        return st, fm, cs

    def debug_normal_equations(self):
        """b = J'^T f, Jacobi scale s, jtj = s^2 colnorm^2 (float32 [U]) and the raw E_g camera sums cam_acc (float32 [33F + 43])."""
        U = 2 * self.n + 6 * self.F + 9
        b, s, jtj = np.empty(U, np.float32), np.empty(U, np.float32), np.empty(U, np.float32)
        cam = np.empty(33 * self.F + 43, np.float32)
        self._check(self.L.i3d_debug_get_normal_equations(self.h, _p(b, C.c_float), _p(s, C.c_float), _p(jtj, C.c_float), _p(cam, C.c_float)))
        return dict(b=b, s=s, jtj=jtj, cam_acc=cam)

    def debug_apply_operator(self, v):
        """q = S (J^T W J) S v for the rows of the last iteration (float32 [U]), through the production operator kernels."""
        U = 2 * self.n + 6 * self.F + 9
        v = np.ascontiguousarray(v, np.float32)
        assert v.shape == (U,)
        q = np.empty(U, np.float32)
        self._check(self.L.i3d_debug_apply_operator(self.h, _p(v, C.c_float), _p(q, C.c_float)))
        return q


def shard_range(n: int, rank: int, world: int, align: int = 512):
    """Voxel index range [begin, end) whose residual rows `rank` owns: equal contiguous ranges of the grid's
    iteration order (8^3-brick-major => z-slabs of bricks), aligned to whole bricks where possible."""
    if world <= 1:
        return 0, n
    per = -(-n // world)
    per = -(-per // align) * align
    b = min(n, rank * per)
    e = min(n, (rank + 1) * per)
    if rank == world - 1:
        e = n
    return b, e


def cut_ranges(cost, world: int, align: int = 64):
    """Cuts the index range [0, n) of a per-voxel cost vector (torch tensor, any device) into `world` contiguous ranges of (nearly) equal
    summed cost; every interior cut is rounded to a multiple of `align` voxels and the cuts are monotone.  Pure function of its input:
    every rank that passes the same (all-reduced) cost vector gets the same ranges."""
    import torch
    n = int(cost.shape[0])
    c = torch.cumsum(cost.to(torch.float64), 0)
    total = float(c[-1].item()) if n > 0 else 0.0
    cuts = [0]
    for r in range(1, world):
        i = int(torch.searchsorted(c, torch.tensor([total * r / world], device=c.device, dtype=c.dtype)).item())
        i = min(n, max(cuts[-1], (i + align // 2) // align * align))
        cuts.append(i)
    cuts.append(n)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def balanced_shard_ranges(eng, dist, params, n: int, align: int = 64, voxel_weight: float = 2.0):
    """Voxel index ranges [begin, end) per rank that balance the WORK rather than the voxel count: one residual build with the
    equal-count split (shard_range) gives, per voxel, the number of valid E_g rows; the cost model rows + voxel_weight * active is
    summed over ranks and cut into `world` equal parts (aligned to `align` voxels).  Call once per grid; returns a list of
    (begin, end) identical on every rank.  (z-slabs of a closed surface see very different numbers of frames: the equal-count
    split left the slowest rank with 1.7x the mean k_eg_apply time at 8 GPUs, profiles/r01 scaling table.)"""
    import torch
    world = dist.get_world_size()
    rank = dist.get_rank()
    eng.set_shard(*shard_range(n, rank, world))
    p = type(params).from_buffer_copy(bytes(params))
    p.build_only = 1
    eng.gn_iteration(p)
    rows = eng.debug_rows(want_jac=False)
    K = int(p.num_observations)
    stride = len(rows["frame"]) // max(K, 1)
    cost = np.zeros(n, np.float64)
    vox = rows["voxel"][:stride]
    valid = (rows["frame"].reshape(K, stride) >= 0).sum(0)
    m = vox >= 0
    cost[vox[m]] = valid[m] + voxel_weight
    t = torch.from_numpy(cost).cuda()
    dist.all_reduce(t)
    ranges = cut_ranges(t, world, align)
    if os.environ.get("I3D_SHARD", "balanced") != "timed":
        return ranges
    return rebalance_by_time(eng, dist, params, n, ranges, t, align)


TIMED_KERNELS = ("k_select_obs", "k_eg_build", "k_eg_accum", "k_eg_cost", "k_eg_apply", "k_op_partial", "k_cg_update", "k_cg_dir")


def rebalance_by_time(eng, dist, params, n, ranges, cost, align=64, rounds=2):
    """Second stage of the shard balance (I3D_SHARD=timed): the row-count model misses per-voxel differences the kernels see (the
    observation selection visits more frames for some slabs of a closed surface than for others).  One full GN iteration per round is
    timed per kernel on every rank (compute kernels only: the exchange kernels contain the waiting for the slowest rank), the model
    cost of every voxel is scaled by (measured time / model cost) of the rank that ran it, and the ranges are cut again.  The engine
    state is restored afterwards.  `cost`: the summed model cost per voxel (device tensor)."""
    import torch
    world, rank = dist.get_world_size(), dist.get_rank()
    saved = eng.download_state()
    p = type(params).from_buffer_copy(bytes(params))
    cost = cost.clone()
    for _ in range(rounds):
        eng.set_shard(*ranges[rank])
        eng.set_kernel_timers(1)
        eng.gn_iteration(p)                      # warm-up (launch attributes, first-touch)
        eng.upload_voxel_params(saved["sdf_refined"], saved["albedo"]); eng.set_camera(saved["poses"], saved["intr"], saved["dist"])
        eng.gn_iteration(p)
        mine = sum(eng.phase_ms(k) for k in TIMED_KERNELS)
        eng.set_kernel_timers(0)
        eng.upload_voxel_params(saved["sdf_refined"], saved["albedo"]); eng.set_camera(saved["poses"], saved["intr"], saved["dist"])
        tt = torch.zeros(world, device="cuda", dtype=torch.float64)
        tt[rank] = mine
        dist.all_reduce(tt)
        c = torch.cumsum(cost, 0)
        scale = torch.ones(world, device="cuda", dtype=torch.float64)
        for r, (b, e_) in enumerate(ranges):
            model = float((c[e_ - 1] - (c[b - 1] if b > 0 else 0.0)).item()) if e_ > b else 0.0
            if model > 0.0 and float(tt[r].item()) > 0.0:
                scale[r] = tt[r] / model
        for r, (b, e_) in enumerate(ranges):
            cost[b:e_] *= scale[r]
        ranges = cut_ranges(cost, world, align)
    return ranges


def _comm_init(self, rank: int, world: int, dist=None):
    """Creates the engine's NCCL communicator.  The 128-byte unique id is produced on rank 0 by the library and
    distributed with torch.distributed (`dist`, already initialised)."""
    if world <= 1:
        return
    import torch
    buf = (C.c_uint8 * 128)()
    if rank == 0:
        if self.L.i3d_comm_unique_id(buf) != 0:
            raise RuntimeError("i3d_comm_unique_id failed: " + self.L.i3d_last_error(None).decode())
    dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
    t = torch.tensor(list(buf), dtype=torch.uint8, device=dev)
    dist.broadcast(t, 0)
    raw = bytes(t.cpu().tolist())
    arr = (C.c_uint8 * 128).from_buffer_copy(raw)
    self._check(self.L.i3d_comm_init(self.h, C.c_int32(rank), C.c_int32(world), arr))
    self.rank, self.world = rank, world
    # peer-memory exchange: every rank maps every peer's mailbox (CUDA IPC).  I3D_XCHG=nccl keeps the ncclAllReduce path.
    self.p2p = False
    if os.environ.get("I3D_XCHG", "p2p") != "nccl" and dist.get_backend() == "nccl":
        mine = (C.c_uint8 * 64)()
        self._check(self.L.i3d_comm_p2p_export(self.h, mine))
        t = torch.tensor(list(mine), dtype=torch.uint8, device="cuda")
        allh = torch.empty(64 * world, dtype=torch.uint8, device="cuda")
        dist.all_gather_into_tensor(allh, t)
        rawh = bytes(allh.cpu().tolist())
        harr = (C.c_uint8 * (64 * world)).from_buffer_copy(rawh)
        rc = self.L.i3d_comm_p2p_connect(self.h, harr)
        ok = torch.tensor([1 if rc == 0 else 0], device="cuda")
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if ok.item() != 1:
            raise RuntimeError("i3d_comm_p2p_connect failed on some rank (" + self.L.i3d_last_error(self.h).decode() + "); set I3D_XCHG=nccl to use ncclAllReduce")
        self.p2p = True


def _set_shard(self, begin: int, end: int):
    self._check(self.L.i3d_set_shard(self.h, C.c_int64(begin), C.c_int64(end)))


Engine.comm_init = _comm_init
Engine.set_shard = _set_shard
