#!/usr/bin/env python
"""bench.py — Gauss-Newton iterations/sec of the joint-refinement hot path (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload c3|c2|c5|small|tiny] [--impl ours|reference]

One "step" = one outer Gauss-Newton iteration of Optimizer::optimize (observation selection,
residual + Jacobian build, weight normalisation, one accepted LM step incl. all PCG iterations and
cost evaluations, parameter update) on the synthetic 2M-voxel / 200-frame hashed-SDF scene (C3).
`value`   : steps/s with every input resident in HBM (whole job, all ranks; device-bracketed wall time, max over ranks).
`e2e`     : the same metric through the C-ABI with HOST (pinned) buffers in the call shape of the reference API,
            Optimizer::optimize: upload grid + frames + camera + SH, `iterations` (10) GN iterations with the lambda ramps,
            download the refined state — every call, inside the timed region.  `e2e.per_iteration_upload` is the conservative
            variant that re-uploads everything before EVERY iteration.
`roofline`: dominant kernel (k_eg_apply, the fused CGNR operator over the E_g rows) and, as `roofline_jacobian_build`, the
            Jacobian-build kernel north_star names: algorithmic bytes of THIS rank / CUDA-event time of THIS rank against the
            measured HBM peak.
`cpu_baseline`: the CPU oracle (float64 restatement of the reference + Ceres semantics) timed on this box's cores on the
            FULL workload (one GN iteration), next to `parity_check`: engine vs oracle on a z-slab of the same scene.
`--impl reference`: the same oracle with all host threads on the full workload (`--ref-max-steps` clips the steps).
Under torchrun (N > 1) voxels are sharded across ranks (one process per GPU); `mg_selfcheck` compares the sharded engine
with an unsharded one on the same GPU after 3 iterations.
`--workload c5`: BASELINE config 5, the coarse-to-fine schedule of Intrinsic3D::refine (0.5M -> 2M -> 8M voxels, 500 frames);
a step is one whole refinement (50 GN iterations + lighting, recolouring, pruning, upsampling), value = GN iterations/s.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = {
    "c3": "synthetic 2M-voxel hashed SDF (bumpy sphere, band 3 voxels @2mm), 200 frames 640x480, per-voxel varying SH (9 coeffs), K=5 observations, all four cost terms",
    "c2": "synthetic 500K-voxel hashed SDF, 50 frames 640x480, K=5, all four cost terms",
    "c5": "coarse-to-fine Intrinsic3D::refine schedule: 3 grid levels 0.5M -> ~2M -> ~8M voxels (4/2/1 mm), 500 frames 640x480 (3 pyramid levels on the coarsest grid), 5 optimize() calls x 10 GN iterations, SVSH lighting + recolouring per call, pruning + x2 upsampling between levels",
    "small": "synthetic 30K-voxel hashed SDF, 8 frames 320x240 (plumbing)",
    "tiny": "synthetic 8K-voxel hashed SDF, 6 frames 160x120 (plumbing)",
}
ITERATIONS = 10   # Optimizer::Config::iterations (data/intrinsic3d.yml): lambda ramp length
KSTAT_KEYS = ("k_eg_apply", "k_eg_build", "k_eg_accum", "k_eg_cost", "k_op_partial", "exchange", "k_cg_dir", "k_cg_update", "k_select_obs",
              "select", "build", "solve", "pcg", "candidate", "total", "launches", "host_syncs")
N_KERNEL_KEYS = 9


def lambda_schedule(p, it):
    """computeVaryingLambda (cost.h:130-143) with data/intrinsic3d.yml: lambda_r 80->10, lambda_s 120->10."""
    k = it % ITERATIONS
    p.lambda_[0] = 0.2
    p.lambda_[1] = 80.0 + (10.0 - 80.0) / (ITERATIONS - 1) * k
    p.lambda_[2] = 120.0 + (10.0 - 120.0) / (ITERATIONS - 1) * k
    p.lambda_[3] = 0.1


def base_config(workload, n, F):
    """Identical in both arms (the driver compares the dicts): what the workload IS, nothing about how it is run."""
    return {"workload": f"{workload}: {WORKLOADS[workload]}", "voxels": int(n), "frames": int(F), "iterations_schedule": ITERATIONS, "lm_steps": 50,
            "inputs_vs_l2": "E_g Jacobian streamed per PCG iteration is ~0.8 GB >> 50 MB L2 of an H100 (no flush needed)"}


DUMP_LIMIT_BYTES = 64 << 20


def write_outputs(out_dir, arrays):
    """--dump-outputs: <out_dir>/<name>.npy in float32/float64; above DUMP_LIMIT_BYTES the per-voxel arrays keep one seeded row sample
    (indices in sample_rows.npy), so two builds are compared on the same voxels."""
    os.makedirs(out_dir, exist_ok=True)
    arrs = {k: np.ascontiguousarray(v, np.float32 if np.asarray(v).dtype == np.float32 else np.float64) for k, v in arrays.items()}
    total = sum(a.nbytes for a in arrs.values())
    if total > DUMP_LIMIT_BYTES:
        n = max(a.shape[0] for a in arrs.values() if a.ndim)
        long_ = [k for k, a in arrs.items() if a.ndim and a.shape[0] == n]
        per_row = sum(arrs[k].nbytes // n for k in long_) + 8
        m = min(n, (DUMP_LIMIT_BYTES - (total - sum(arrs[k].nbytes for k in long_)) - 4096) // per_row)
        rows = np.sort(np.random.default_rng(0).choice(n, m, replace=False))
        for k in long_:
            arrs[k] = np.ascontiguousarray(arrs[k][rows])
        arrs["sample_rows"] = rows.astype(np.float64)
    for k, a in arrs.items():
        np.save(os.path.join(out_dir, f"{k}.npy"), a)


def iteration_outputs(info):
    """what i3d_gn_iteration returns besides the state"""
    nlm = int(info.lm_iterations)
    return {"cost": [info.cost_initial, info.cost_final], "type_residuals": list(info.type_residuals), "type_costs": list(info.type_costs),
            "step_accepted": [info.step_accepted], "cg_iterations": list(info.cg_iterations)[:nlm]}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled during the timed region."""
    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index=0):
        self.samples = []
        self.proc = None
        self.index = index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.samples.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        mhz, mx, reasons = [], [], set()
        for ln in self.samples:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 6:
                continue
            try:
                mhz.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[2:6]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(mhz) if mhz else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(mhz), "window": "warm-up + timed steps"}


_COLOR_CACHE = {}


def color_frames_once(scene):
    """Synthetic B,G,R frames for the recolouring legs, generated once per process."""
    if "c" not in _COLOR_CACHE:
        from intrinsic3d_b200.scene import make_color_frames
        _COLOR_CACHE["c"] = make_color_frames(scene)
    return _COLOR_CACHE["c"]


def make_params(scene):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = scene["thres_shell"]
    return p


def slab_scene(scene, fraction):
    """The first `fraction` of the voxels in brick order (a z-slab of the same grid), all frames."""
    n = scene["xyz"].shape[0]
    m = n if fraction >= 1.0 else max(2000, int(n * fraction))
    s = dict(scene)
    for k in ("xyz", "sdf0", "sdf_refined", "albedo", "weight", "rgb", "sh"):
        s[k] = scene[k][:m].copy()
    return s, m


def run_cpu(scene, steps, warmup, threads, parallel_cg):
    """The oracle on the FULL scene: `warmup` untimed + `steps` timed GN iterations of the lambda schedule."""
    from oracle import Oracle
    o = Oracle(threads=threads, parallel_cg=parallel_cg)
    o.load_scene(scene)
    p = make_params(scene)
    times, phases = [], []
    for it in range(warmup + steps):
        if it == warmup and warmup > 0:
            o.load_scene(scene)
        lambda_schedule(p, it - warmup if it >= warmup else it)
        t0 = time.perf_counter()
        info = o.gn_iteration(p)
        dt = time.perf_counter() - t0
        if it >= warmup:
            times.append(dt)
            phases.append((info.time_add, info.time_build, info.time_solve, info.cg_iterations_total, info.lm_iterations))
    t_step = sum(times) / len(times)
    return dict(s_per_step=t_step, value=1.0 / t_step, step_s=times,
                time_add=sum(x[0] for x in phases) / len(phases), time_build=sum(x[1] for x in phases) / len(phases),
                time_solve=sum(x[2] for x in phases) / len(phases), cg_iterations=[x[3] for x in phases], lm_iterations=[x[4] for x in phases])


def parity_check(scene, fraction, device, threads):
    """Engine vs oracle on the same z-slab of the benchmark scene (all frames): one full GN iteration from identical inputs.
    Gate = SURVEY.md §8(d) 'parity gate'.  Returns a dict with the achieved bounds and `ok`."""
    from intrinsic3d_b200.engine import Engine
    from oracle import Oracle
    s, m = slab_scene(scene, fraction)
    K = 5
    p = make_params(scene)
    lambda_schedule(p, 0)
    e = Engine(device)
    e.load_scene(s)
    o = Oracle(threads=threads, parallel_cg=True)
    o.load_scene(s)
    # rows at the initial point
    p.build_only = 1
    ie, io = e.gn_iteration(p), o.gn_iteration(p)
    fe, we, ae = e.debug_observations(K)
    fo, wo, ao = o.observations(K)
    sel_exact = bool(np.array_equal(ae, ao) and np.array_equal(fe, fo) and np.array_equal(we.view(np.uint32), wo.view(np.uint32)))
    re_, ro = e.debug_rows(want_jac=True), o.rows(0)
    me = {(int(v), int(f)): i for i, (v, f) in enumerate(zip(re_["voxel"], re_["frame"])) if f >= 0}
    mo = {(int(v), int(f)): i for i, (v, f) in enumerate(zip(ro["voxel"], ro["aux"])) if f >= 0}
    same_rows = set(me) == set(mo)
    res_rel, jac_rel = None, None
    if same_rows and mo:
        keys = list(mo)
        ie_idx = np.array([me[k] for k in keys]); io_idx = np.array([mo[k] for k in keys])
        res_e, res_o = re_["residual"][ie_idx], ro["residual"][io_idx]
        res_rel = float(np.max(np.abs(res_e - res_o) / np.abs(res_o)))
        Jo = o.eg_jacobian()[io_idx]
        Je = re_["J"][:, ie_idx].T.astype(np.float64)
        jac_rel = float(np.max(np.abs(Je - Jo) / np.abs(Jo).max(axis=1, keepdims=True)))
    counts_equal = list(ie.type_residuals) == list(io.type_residuals) and ie.num_active == io.num_active
    cost_rel = abs(ie.cost_initial - io.cost_initial) / abs(io.cost_initial)
    # the full step (natural PCG termination)
    p.build_only = 0
    e.load_scene(s); o.load_scene(s)
    ie, io = e.gn_iteration(p), o.gn_iteration(p)
    nlm = io.lm_iterations
    cg_equal = ie.lm_iterations == io.lm_iterations and list(ie.cg_iterations)[:nlm] == list(io.cg_iterations)[:nlm]
    se, so = e.debug_step()[0], o.step()[0]
    nv = m
    F = s["poses"].shape[0]
    step_rel = {}
    for name, lo, hi in (("sdf", 0, nv), ("albedo", nv, 2 * nv), ("poses", 2 * nv, 2 * nv + 6 * F), ("intrinsics", 2 * nv + 6 * F, 2 * nv + 6 * F + 4),
                         ("distortion", 2 * nv + 6 * F + 4, 2 * nv + 6 * F + 9)):
        ref = float(np.abs(so[lo:hi]).max())
        step_rel[name] = float(np.abs(se[lo:hi] - so[lo:hi]).max() / ref) if ref > 0 else 0.0
    # camera blocks on a partial grid (fraction < 1) are constrained by a fraction of their rows only: 5e-3 there, 1e-3 on a whole grid
    cam_tol = 1e-3 if fraction >= 1.0 else 5e-3
    step_ok = all(v <= (1e-3 if k in ("sdf", "albedo") else cam_tol) for k, v in step_rel.items())
    ok = bool(sel_exact and same_rows and counts_equal and res_rel is not None and res_rel <= 1e-4 and jac_rel <= 1e-3 and cost_rel <= 1e-9 and cg_equal
              and ie.step_accepted == io.step_accepted and step_ok)
    e.close()
    return {"ok": ok, "sample": f"first {m} of {scene['xyz'].shape[0]} voxels in brick order (z-slab), all {F} frames, K={K}",
            "selection_bit_exact": sel_exact, "same_row_set": bool(same_rows), "row_counts_equal": bool(counts_equal), "eg_rows": int(io.type_residuals[0]),
            "residual_max_rel": res_rel, "jacobian_max_rel_of_row_max": jac_rel, "cost_initial_rel": float(cost_rel), "cg_iterations_equal": bool(cg_equal),
            "cg_iterations": [int(x) for x in list(io.cg_iterations)[:nlm]], "accepted": [int(ie.step_accepted), int(io.step_accepted)],
            "step_max_rel_of_block_max": step_rel, "gate": f"selection bit-exact; residual <= 1e-4; J <= 1e-3 of row max; equal CG counts; step <= 1e-3 of the block max for sdf/albedo, <= {cam_tol:g} for the camera blocks (SURVEY §8d; the slab sample constrains the 200 poses weakly)"}


def reference_arm(args, ncores):
    """bench.py --impl reference: the reference's CPU path (oracle port; Ceres itself cannot be built offline) on the FULL workload."""
    import torch
    from intrinsic3d_b200.scene import config_scene
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    wl = "c3" if args.workload == "c5" else args.workload
    scene = config_scene(wl, device=dev)
    n, F = scene["xyz"].shape[0], scene["lum"].shape[0]
    # The restated path stops scaling well before 128 threads (32 threads were fastest on a 128-core host)
    threads = min(ncores, 32)
    steps = max(1, args.steps if args.ref_max_steps is None else min(args.steps, args.ref_max_steps))
    warmup = min(args.warmup, 1)
    r = run_cpu(scene, steps, warmup, threads, parallel_cg=True)
    sample = (f"FULL workload ({n} voxels, {F} frames), one GN iteration per step; {steps} timed + {warmup} warm-up "
              f"(requested {args.steps} + {args.warmup})")
    line = {"impl": "reference", "metric": "gauss_newton_iterations_per_sec", "value": r["value"], "unit": "GN iter/s", "n_gpus": args.gpus,
            "steps": steps, "warmup": warmup, "steps_requested": args.steps, "warmup_requested": args.warmup,
            "ms_per_step": 1e3 * r["s_per_step"], "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f64", "data": "synthetic", "config": base_config(wl, n, F),
            "precision": "float64 throughout (Ceres semantics restated)", "parallelism": f"{threads} host threads",
            "cpu_baseline": {"value": r["value"], "unit": "GN iter/s", "cores": threads, "kind": "port", "sample": sample,
                             "s_per_step": r["s_per_step"], "step_s": r["step_s"], "time_add": r["time_add"], "time_solve": r["time_solve"], "cg_iterations": r["cg_iterations"],
                             "note": "oracle = float64 restatement of the reference + Ceres 2.1 semantics (Ceres/Eigen/OpenCV unavailable offline); all host threads incl. a threaded CGNR (more generous than Ceres 2.1's serial CGNR)"},
            "e2e": {"value": r["value"], "unit": "GN iter/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", default=os.environ.get("I3D_WORKLOAD", "c3"), choices=sorted(WORKLOADS))
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--parity-fraction", type=float, default=1.0 / 16.0)
    ap.add_argument("--ref-max-steps", type=int, default=None, help="--impl reference: clip the timed steps (a full-C3 CPU iteration takes ~15 s)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-parity-check", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--e2e-steps", type=int, default=3)
    ap.add_argument("--no-lighting", action="store_true")
    ap.add_argument("--no-selfcheck", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (refined state + iteration info) as DIR/<name>.npy")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    ncores = os.cpu_count() or 1

    # ------------------------------------------------------------------ reference arm (CPU oracle)
    if args.impl == "reference":
        if rank != 0:
            return
        reference_arm(args, ncores)
        return

    import torch
    from intrinsic3d_b200.scene import config_scene

    # ------------------------------------------------------------------ our arm
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the engine has no CPU fallback")
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist_mod
        dist = dist_mod
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    if args.workload == "c5":
        import bench_c5
        outputs = bench_c5.run(args, rank, world, local_rank, dist, ClockSampler)
        if args.dump_outputs and outputs is not None:
            write_outputs(args.dump_outputs, outputs)
        return
    from intrinsic3d_b200.engine import Engine, shard_range

    scene = config_scene(args.workload, device=f"cuda:{local_rank}")
    n = scene["xyz"].shape[0]
    F = scene["lum"].shape[0]
    config = base_config(args.workload, n, F)
    eng = Engine(local_rank)
    if world > 1:
        eng.comm_init(rank, world, dist)
    eng.load_scene(scene)
    p = make_params(scene)
    my_range = (0, n)
    shard_ranges = None
    if world > 1:
        # equal WORK per rank (E_g rows + active voxels from one residual build), not equal voxel counts; I3D_SHARD=equal keeps the latter
        if os.environ.get("I3D_SHARD", "balanced") == "equal":
            shard_ranges = [shard_range(n, r, world) for r in range(world)]
        else:
            from intrinsic3d_b200.engine import balanced_shard_ranges
            lambda_schedule(p, 0)
            shard_ranges = balanced_shard_ranges(eng, dist, p, n)
        my_range = shard_ranges[rank]
        eng.set_shard(*my_range)

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        if dist is None:
            return x
        t = torch.tensor([x], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def reset_state():
        eng.upload_voxel_params(scene["sdf_refined"], scene["albedo"])
        eng.set_camera(scene["poses"], scene["intr"], scene["dist"])

    # nvidia-smi needs ~0.2 s to start producing samples and the timed region can be shorter than that: the sampler runs from
    # before the warm-up steps (same workload) through the timed region
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
        time.sleep(0.3)
    for it in range(args.warmup):
        lambda_schedule(p, it)
        eng.gn_iteration(p)
    reset_state()
    infos, kstats = [], []
    barrier()
    t0 = time.perf_counter()
    for it in range(args.steps):
        lambda_schedule(p, it)
        info = eng.gn_iteration(p)
        infos.append(info)
        kstats.append({k: (eng.phase_ms(k), eng.phase_count(k)) for k in KSTAT_KEYS})
    barrier()
    elapsed = max_over_ranks(time.perf_counter() - t0)
    clocks = sampler.stop() if rank == 0 else None
    value = args.steps / elapsed
    if args.dump_outputs and rank == 0 and infos:
        write_outputs(args.dump_outputs, {**eng.download_state(), **iteration_outputs(infos[-1])})
    # per-kernel table: ONE extra, untimed step with an event pair around every kernel (in the timed region only the phases, the
    # two roofline kernels k_eg_rows / k_eg_apply and k_select_obs carry events: an event between two kernels suppresses their
    # programmatic-dependent-launch overlap)
    eng.set_kernel_timers(1)
    lambda_schedule(p, min(3, args.steps - 1))
    eng.gn_iteration(p)
    detail = {k: (eng.phase_ms(k), eng.phase_count(k)) for k in KSTAT_KEYS}
    eng.set_kernel_timers(0)

    # ------------------------------------------------------------------ roofline: THIS rank's algorithmic bytes / THIS rank's kernel time
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak_gbs = float(peaks.get("hbm_gbs", 3350.0))
    peak_src = "measured (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks else "data sheet 3350 GB/s (H100 SXM HBM3, not measured)"
    U = 2 * n + 6 * F + 9
    K = p.num_observations
    # rows / active voxels this rank owns (I3DIterInfo carries the GLOBAL sums when sharded)
    rows_dbg = eng.debug_rows(want_jac=False)
    local_rows = int((rows_dbg["frame"] >= 0).sum())
    local_active = int(len(rows_dbg["frame"]) // K) if K else 0          # slots per k (stride, multiple of 64)
    b0, b1 = my_range
    local_unknowns = 2 * (b1 - b0) + 6 * F + 9
    W_, H_ = scene["lum"].shape[2], scene["lum"].shape[1]

    def kernel_roofline(name, bytes_per_launch, formula):
        tot_ms = sum(k[name][0] for k in kstats)
        cnt = sum(k[name][1] for k in kstats)
        if cnt == 0 or tot_ms == 0:
            return None
        ach = bytes_per_launch / (tot_ms / cnt * 1e-3) / 1e9
        return {"kernel": name, "bound": "hbm", "achieved": ach, "peak": peak_gbs, "unit": "GB/s", "frac": ach / peak_gbs, "peak_source": peak_src,
                "bytes_per_launch": bytes_per_launch, "bytes_formula": formula, "avg_launch_ms": tot_ms / cnt, "launches_timed": cnt,
                "timing": "CUDA events on the engine stream inside the timed region",
                "scope": f"rank 0 of {world}: rows and time of this rank only"}

    traffic = {}
    try:
        traffic = json.load(open(os.path.join(ROOT, "profiles", "traffic.json")))
    except Exception:
        pass
    roof_apply = kernel_roofline("k_eg_apply", local_rows * 124 + local_active * 40 + local_unknowns * 12,
                                 "R_g*124 (29 J floats + weight + frame id) + N_a*40 (index + 9 neighbour ids) + U*12 (read ps, read-modify-write qg)")
    img_bytes = min(F * W_ * H_ * 4, local_rows * 256)
    roof_build = kernel_roofline("k_eg_build", local_active * (16 + 36 + 8 * K) + local_rows * 124 + img_bytes,
                                 "SURVEY.md §8(d) B_k2 = N_a*(16+36+8K) + R_g*(29*4+4+4) + U_img, U_img = min(F*W*H*4, R_g*256)")
    for r_, key in ((roof_apply, "k_eg_apply"), (roof_build, "k_eg_build")):
        if r_ is not None:
            t_ = traffic.get(key) or {}
            r_["traffic"] = t_.get("dram_bytes_per_launch") if world == 1 else None
            r_["traffic_source"] = t_.get("source") if world == 1 else "ncu capture is single-GPU (full C3 grid); not applicable to a shard"

    # per-rank means of the kernel / phase times (load balance across the shards): [world][len(keys)]
    per_rank = None
    if world > 1:
        keys_pr = KSTAT_KEYS[:N_KERNEL_KEYS] + ("select", "build", "pcg", "candidate", "total")
        mine = torch.tensor([float(detail[k][0]) if k in KSTAT_KEYS[:N_KERNEL_KEYS] else float(np.mean([s_[k][0] for s_ in kstats])) for k in keys_pr],
                            device="cuda", dtype=torch.float64)
        allr = torch.empty(world * len(keys_pr), device="cuda", dtype=torch.float64)
        dist.all_gather_into_tensor(allr, mine)
        allr = allr.view(world, len(keys_pr)).cpu().numpy()
        per_rank = {k: [round(float(x), 3) for x in allr[:, i]] for i, k in enumerate(keys_pr)}

    # ------------------------------------------------------------------ multi-GPU self-check: sharded vs unsharded engine, same GPU, 3 iterations
    mg_selfcheck = None
    if world > 1 and not args.no_selfcheck:
        ref = Engine(local_rank)
        ref.load_scene(scene)
        reset_state()
        ok, log = True, []
        for it in range(3):
            lambda_schedule(p, it)
            a, b = eng.gn_iteration(p), ref.gn_iteration(p)
            sa, sb = eng.download_state(), ref.download_state()
            step = ref.debug_step()[0]
            nlm = b.lm_iterations
            chk = dict(rows=list(a.type_residuals) == list(b.type_residuals), active=a.num_active == b.num_active,
                       cost0=abs(a.cost_initial - b.cost_initial) <= 1e-9 * abs(b.cost_initial),
                       cg=list(a.cg_iterations)[:a.lm_iterations] == list(b.cg_iterations)[:nlm], accepted=a.step_accepted == b.step_accepted,
                       cost1=abs(a.cost_final - b.cost_final) <= 1e-5 * abs(b.cost_final),
                       sdf=float(np.abs(sa["sdf_refined"] - sb["sdf_refined"]).max()) <= 1e-3 * float(np.abs(step[:n]).max()),
                       poses=float(np.abs(sa["poses"] - sb["poses"]).max()) <= 1e-3 * max(float(np.abs(step[2 * n:2 * n + 6 * F]).max()), 1e-30))
            log.append({k: bool(v) for k, v in chk.items()})
            ok = ok and all(chk.values())
            # identical inputs for the next iteration on every engine (the unsharded run is not bitwise reproducible between GPUs: float atomics)
            for k in ("sdf_refined", "albedo", "poses", "intr", "dist"):
                t = torch.from_numpy(sb[k]).cuda()
                dist.broadcast(t, 0)
                sb[k] = t.cpu().numpy()
            for en in (eng, ref):
                en.upload_voxel_params(sb["sdf_refined"], sb["albedo"])
                en.set_camera(sb["poses"], sb["intr"], sb["dist"])
        t = torch.tensor([1 if ok else 0], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        mg_selfcheck = {"ok": bool(t.item() == 1), "iterations": 3, "rank0_checks": log,
                        "what": "voxel-sharded engine vs an unsharded engine on the same GPU and inputs: row counts, cost, PCG iteration counts, accept decision, state within 1e-3 of the step"}
        ref.close()
        reset_state()

    # ------------------------------------------------------------------ e2e: host buffers through the C-ABI
    e2e = None
    if not args.no_e2e:
        keys = ("xyz", "sdf0", "sdf_refined", "albedo", "weight", "rgb", "lum", "depth", "poses", "intr", "dist", "sh")
        pinned = {}
        for k in keys:
            a = np.ascontiguousarray(scene[k])
            pinned[k] = torch.from_numpy(a.copy()).pin_memory()
        host = {k: v.numpy() for k, v in pinned.items()}
        h2d = sum(host[k].nbytes for k in keys)

        def upload_all():
            eng.upload_grid(host["xyz"], host["sdf0"], host["sdf_refined"], host["albedo"], host["weight"], host["rgb"], scene["voxel_size"])
            eng.upload_frames(host["lum"], host["depth"], 1.0)
            eng.set_camera(host["poses"], host["intr"], host["dist"])
            eng.set_sh(host["sh"])
            if world > 1:
                eng.set_shard(*my_range)

        # the call a user of the reference makes: Optimizer::optimize with `iterations` = 10 (data/intrinsic3d.yml)
        def optimize_call():
            upload_all()
            for it in range(ITERATIONS):
                lambda_schedule(p, it)
                eng.gn_iteration(p)
            return eng.download_state()

        out = optimize_call()
        d2h = sum(v.nbytes for v in out.values())
        barrier()
        t2 = time.perf_counter()
        ncalls = max(1, args.e2e_steps)
        for _ in range(ncalls):
            optimize_call()
        barrier()
        el2 = max_over_ranks(time.perf_counter() - t2)
        e2e = {"value": ncalls * ITERATIONS / el2, "unit": "GN iter/s", "h2d_bytes_per_step": int(h2d // ITERATIONS), "d2h_bytes_per_step": int(d2h // ITERATIONS),
               "definition": "Optimizer::optimize call shape: per call, upload grid+frames+camera+SH from pinned host memory, 10 GN iterations (lambda ramps), download the refined state; bytes per step = bytes per call / 10",
               "iterations_per_call": ITERATIONS, "calls": ncalls, "h2d_bytes_per_call": int(h2d), "d2h_bytes_per_call": int(d2h), "ms_per_call": 1e3 * el2 / ncalls}

        # conservative variant: everything re-uploaded before EVERY iteration
        def e2e_step(it):
            lambda_schedule(p, it)
            upload_all()
            eng.gn_iteration(p)
            return eng.download_state()

        e2e_step(0)
        barrier()
        t1 = time.perf_counter()
        for it in range(args.e2e_steps):
            e2e_step(it)
        barrier()
        el = max_over_ranks(time.perf_counter() - t1)
        e2e["per_iteration_upload"] = {"value": args.e2e_steps / el, "unit": "GN iter/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h), "steps": args.e2e_steps,
                                       "note": "each step = upload grid+frames+camera+SH, ONE GN iteration, download refined state (PCIe-bound: the 492 MB of frames never change)"}

        # one whole refinement level of Intrinsic3D::refine through the C-ABI with host buffers: upload (grid, frames, colour frames,
        # camera), thin-shell pruning, SVSH lighting estimate, the 10 GN iterations, recolouring, download of the refined grid and camera.
        if world == 1 and not args.no_lighting:
            try:
                from intrinsic3d_b200.engine import default_lighting_params
                col_t = torch.from_numpy(color_frames_once(scene)).pin_memory()
                col_host = col_t.numpy()
                LPl = default_lighting_params()
                LPl.thres_shell = scene["thres_shell"]

                def refine_level():
                    eng.upload_grid(host["xyz"], host["sdf0"], host["sdf_refined"], host["albedo"], host["weight"], host["rgb"], scene["voxel_size"])
                    eng.upload_frames(host["lum"], host["depth"], 1.0)
                    eng.upload_color_frames(col_host)
                    eng.set_camera(host["poses"], host["intr"], host["dist"])
                    eng.clear_voxels_outside_thin_shell(float(scene["thres_shell"]))
                    li = eng.estimate_lighting(LPl)
                    for it in range(ITERATIONS):
                        lambda_schedule(p, it)
                        eng.gn_iteration(p)
                    cnt = eng.recompute_colors(0.02, 5)
                    g = eng.download_grid()
                    st = eng.download_state()
                    return li, cnt, g, st
                refine_level()
                t3 = time.perf_counter()
                li, cnt, g, st = refine_level()
                el3 = time.perf_counter() - t3
                e2e["refine_level_call"] = {
                    "ms_per_call": 1e3 * el3, "value": ITERATIONS / el3, "unit": "GN iter/s",
                    "steps": "upload grid+frames+colour+camera, clear_voxels_outside_thin_shell, estimate_lighting, 10 gn_iteration, recompute_colors, download grid+camera",
                    "h2d_bytes_per_call": int(h2d - host["sh"].nbytes + col_host.nbytes), "d2h_bytes_per_call": int(sum(v.nbytes for v in g.values() if hasattr(v, "nbytes")) + sum(v.nbytes for v in st.values())),
                    "voxels_in": int(n), "voxels_after_pruning": int(len(g["xyz"])), "subvolumes": int(li.num_subvolumes), "voxels_recolored": int(cnt[0])}
                # restore the benchmark grid for the legs below
                eng.upload_grid(host["xyz"], host["sdf0"], host["sdf_refined"], host["albedo"], host["weight"], host["rgb"], scene["voxel_size"])
                eng.set_sh(host["sh"])
            except Exception as ex:
                e2e["refine_level_call"] = {"error": str(ex)}

    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return

    # ------------------------------------------------------------------ CPU legs (rank 0, N = 1 only): full-workload baseline + slab parity check
    cpu_baseline, parity = None, None
    if world == 1 and not args.no_cpu_baseline:
        r = run_cpu(scene, 1, 0, min(8, ncores), parallel_cg=False)
        cpu_baseline = {"value": r["value"], "unit": "GN iter/s", "cores": min(8, ncores), "kind": "port",
                        "sample": f"FULL workload ({n} voxels, all {F} frames), ONE GN iteration (the first of the lambda schedule), no extrapolation",
                        "s_per_step": r["s_per_step"], "time_add": r["time_add"], "time_build": r["time_build"], "time_solve": r["time_solve"],
                        "cg_iterations": r["cg_iterations"],
                        "note": "reference-equivalent CPU path: float64 oracle restating the reference + Ceres 2.1.0 semantics (Ceres unavailable offline); 8 threads for Jacobian/cost evaluation (num_threads = 8, nls_solver.cpp:333), serial CGNR like Ceres 2.1"}
    if world == 1 and not args.no_parity_check:
        try:
            parity = parity_check(scene, args.parity_fraction, local_rank, min(32, ncores))
        except Exception as ex:
            parity = {"ok": False, "error": str(ex)}

    # ------------------------------------------------------------------ SVSH lighting (runs once before every optimize() in the reference)
    lighting = None
    if not args.no_lighting and world == 1:
        try:
            from intrinsic3d_b200.engine import default_lighting_params
            LP = default_lighting_params()
            LP.thres_shell = scene["thres_shell"]
            eng.estimate_lighting(LP)
            walls, li = [], None
            for _ in range(5):
                t0 = time.perf_counter()
                li = eng.estimate_lighting(LP)
                walls.append(time.perf_counter() - t0)
            lighting = {"call": "i3d_estimate_lighting (LightingSVSH::estimate + computeVoxelShCoeffs), state resident", "subvolume_size_m": float(LP.subvolume_size),
                        "subvolumes": int(li.num_subvolumes), "data_rows": int(li.num_data_rows), "reg_pairs": int(li.num_reg_pairs),
                        "lm_iterations": int(li.lm_iterations), "cg_iterations": int(li.cg_iterations_total), "usable": int(li.usable),
                        "cost": [float(li.cost_initial), float(li.cost_final)], "wall_ms": 1e3 * float(np.median(walls)),
                        "device_ms": {"accumulate": 1e3 * li.time_accumulate, "solve": 1e3 * li.time_solve, "interpolate": 1e3 * li.time_interpolate}}
        except Exception as ex:      # reported, never fatal for the headline line
            lighting = {"error": str(ex)}

    # ------------------------------------------------------------------ voxel recolouring (Intrinsic3D::recomputeColors, after every optimize())
    recolor = None
    if not args.no_lighting and world == 1:
        try:
            eng.upload_color_frames(color_frames_once(scene))
            eng.recompute_colors(0.02, 5)
            walls, cnt = [], None
            for _ in range(3):
                t0 = time.perf_counter()
                cnt = eng.recompute_colors(0.02, 5)
                walls.append(time.perf_counter() - t0)
            recolor = {"call": "i3d_recompute_colors (SDFColorization::add x F + compute), state and frames resident", "frames": int(F),
                       "voxels_recolored": int(cnt[0]), "observations": int(cnt[1]), "wall_ms": 1e3 * float(np.median(walls)),
                       "device_ms": eng.phase_ms("recolor")}
        except Exception as ex:
            recolor = {"error": str(ex)}

    # ------------------------------------------------------------------ grid-level transition (prepareGridLevel / finishGridLevel); LAST: it changes the grid
    gridops = None
    if not args.no_lighting and world == 1:
        try:
            vs0 = float(scene["voxel_size"])
            steps = []
            for name, fn in (("clear_voxels_outside_thin_shell(2.0 vs)", lambda: eng.clear_voxels_outside_thin_shell(2.0 * vs0)),
                             ("upsample_grid", lambda: eng.upsample_grid()),
                             ("clear_voxels_outside_thin_shell(2.0 vs/2)", lambda: eng.clear_voxels_outside_thin_shell(vs0))):
                n_in = int(eng.n)
                t0 = time.perf_counter()
                n_out = fn()
                wall = time.perf_counter() - t0
                steps.append({"op": name, "voxels_in": n_in, "voxels_out": int(n_out), "wall_ms": 1e3 * wall,
                              "device_ms": eng.phase_ms("upsample" if name.startswith("upsample") else "prune")})
            gridops = {"call": "i3d_clear_voxels_outside_thin_shell / i3d_upsample_grid (SDFAlgorithms), grid resident; wall includes the device hash + neighbour-table rebuild",
                       "steps": steps}
        except Exception as ex:
            gridops = {"error": str(ex)}

    phase_keys = ("select", "build", "pcg", "candidate", "total")
    # device timeline of one iteration ("total": first to last event on the engine stream) vs the wall clock per step: the difference is time
    # the GPU stream was idle between iterations (host-side work of the C-ABI call and of this loop)
    host_gap = 1e3 * elapsed / args.steps - float(np.mean([s["total"][0] for s in kstats]))
    line = {
        "metric": "gauss_newton_iterations_per_sec", "value": value, "unit": "GN iter/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * elapsed / args.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic", "config": config,
        "precision": "state/residuals/reductions f64, Jacobian + PCG vectors f32", "parallelism": f"voxel-sharded x{world}" if world > 1 else "single GPU",
        "shard_ranges": shard_ranges, "exchange": ("peer memory over NVLink (CUDA IPC mailboxes)" if getattr(eng, "p2p", False) else "ncclAllReduce") if world > 1 else None,
        "problem": {"active_voxels": int(infos[0].num_active), "eg_rows": int(infos[0].type_residuals[0]), "parameters": int(infos[0].num_parameters),
                    "rank0_rows": local_rows, "rank0_row_slots_per_k": local_active},
        "clocks": clocks, "e2e": e2e, "gpu_launches": int(sum(k["launches"][1] for k in kstats)),
        "host_syncs_per_step": float(np.mean([k["host_syncs"][1] for k in kstats])),
        "roofline": roof_apply, "roofline_jacobian_build": roof_build, "cpu_baseline": cpu_baseline, "parity_check": parity, "mg_selfcheck": mg_selfcheck,
        "lighting": lighting, "recolor": recolor, "gridops": gridops,
        "per_step": {"cg_iterations": [int(i.cg_iterations_total) for i in infos], "lm_iterations": [int(i.lm_iterations) for i in infos],
                     "accepted": [int(i.step_accepted) for i in infos], "cost_initial": [float(i.cost_initial) for i in infos],
                     "cost_final": [float(i.cost_final) for i in infos],
                     "phase_ms": {k: [round(s[k][0], 3) for s in kstats] for k in phase_keys},
                     "host_gap_ms_mean": round(host_gap, 3),
                     "k_eg_apply_ms": [round(s["k_eg_apply"][0], 3) for s in kstats], "k_eg_build_ms": [round(s["k_eg_build"][0], 3) for s in kstats],
                     "k_eg_cost_ms": [round(s["k_eg_cost"][0], 3) for s in kstats], "k_select_obs_ms": [round(s["k_select_obs"][0], 3) for s in kstats],
                     "kernel_ms_detail_step": {k: [round(detail[k][0], 3), detail[k][1]] for k in KSTAT_KEYS[:N_KERNEL_KEYS]},
                     "kernel_ms_detail_note": "[sum ms, launches] of one extra untimed step with events around every kernel (i3d_debug_set_kernel_timers)",
                     "per_rank_mean_ms": per_rank},
    }
    print(json.dumps(line))
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
