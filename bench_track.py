#!/usr/bin/env python
"""bench_track.py — frame-to-model tracking (i3d_track_sensor_frames) of every frame of a workload against its fused surface, one JSON line.

    python bench_track.py [--workload c3|c2|small|tiny] [--reps 3]

The workload's depth frames go into the sensor store, are fused there at the true poses (i3d_fusion_integrate_sensor), and every frame is
then tracked against sdf0 from the scene's perturbed poses with the default parameters (3 levels, iterations {10, 5, 4}).  Reported, the
median of --reps calls after one warm-up call: device ms of the call (phase "track", CUDA events inside the library) in total and per frame,
and the phases track_predict / track_pyramid / track_icp; from one further call with per-kernel timers, k_track_rows' device time against
the byte model below as a share of 3350 GB/s (H100 SXM HBM3); pose errors against the true poses before and after.  The GPU name and
power limit are read in the same run.  Writes nothing.

Byte model of k_track_rows, per pixel of the level and per iteration: input depth (4 B) and camera-frame normal (12 B), and the gathered
prediction depth (4 B) and world normal (12 B), counted for every pixel (an upper bound: pixels without depth or outside the prediction
read less), plus the 1-byte correspondence mask at level 0.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_GBS = 3350.0


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return out.stdout.strip() or None
    except Exception:
        return None


def rows_bytes(W, H, n, levels, iterations):
    total = 0
    for l in range(levels):
        total += iterations[l] * n * W * H * (32 + (1 if l == 0 else 0))
        W, H = W // 2, H // 2
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import torch
    import track_ref as tr
    from fusion_ref import depth_range, scene_inputs
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene

    gpu = gpu_info()
    s = config_scene(args.workload, device="cuda:0" if torch.cuda.is_available() else "cpu")
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    F, H, W = depth.shape
    e = engine.Engine(0)
    e.sensor_frames_begin(dcam, ccam, F)
    e.sensor_frames_add(depth, bgr)
    p = engine.default_fusion_params()
    p.voxel_size = float(s["voxel_size"])
    p.depth_min, p.depth_max = depth_range(s)
    ids = np.arange(F, dtype=np.int32)
    e.fusion_begin(p)
    e.fusion_integrate_sensor(ids, c2w, w2c)
    voxels = e.fusion_finish()
    true = tr.aa_to_rt(s["poses_true"])
    start = tr.aa_to_rt(s["poses"])
    tp = engine.default_track_params()
    e.track_sensor_frames(ids, start)
    dev, walls, phases, digest = [], [], {k: [] for k in ("track_predict", "track_pyramid", "track_icp")}, None
    for _ in range(max(1, args.reps)):
        t0 = time.perf_counter()
        out, infos = e.track_sensor_frames(ids, start)
        walls.append(1e3 * (time.perf_counter() - t0))
        dev.append(e.phase_ms("track"))
        for k in phases:
            phases[k].append(e.phase_ms(k))
        d = out.tobytes() + repr(infos).encode()
        assert digest is None or d == digest, "tracking not run-to-run identical"
        digest = d
    corr = e.phase_count("track_correspondences")
    e.set_kernel_timers(1)
    e.track_sensor_frames(ids, start)
    rows_ms, rows_launches = e.phase_ms("k_track_rows"), e.phase_count("k_track_rows")
    e.set_kernel_timers(0)
    its = list(tp.iterations)
    nbytes = rows_bytes(W, H, F, tp.num_levels, its)
    r0, t0e = tr.pose_errors(start, true)
    r1, t1e = tr.pose_errors(out, true)
    ms = float(np.median(dev))
    line = {"metric": "track_all_frames_ms", "value": ms, "unit": "ms", "higher_is_better": False, "workload": args.workload, "gpu": gpu,
            "reps": len(dev), "frames": int(F), "size": [int(W), int(H)], "voxels": int(voxels), "device_ms_per_frame": ms / F,
            "wall_ms": float(np.median(walls)), "phases_ms": {k: float(np.median(v)) for k, v in phases.items()},
            "iterations": its[:tp.num_levels], "correspondences": int(corr),
            "status_counts": {str(k): int(sum(1 for i in infos if i["status"] == k)) for k in range(4)},
            "k_track_rows": {"ms": rows_ms, "launches": rows_launches, "model_bytes": nbytes,
                             "gbs": nbytes / (rows_ms * 1e6) if rows_ms > 0 else None,
                             "share_of_hbm": nbytes / (rows_ms * 1e6) / HBM_GBS if rows_ms > 0 else None},
            "pose_error_before": {"rot_deg_median": float(np.median(r0)), "rot_deg_max": float(r0.max()),
                                  "centre_m_median": float(np.median(t0e)), "centre_m_max": float(t0e.max())},
            "pose_error_after": {"rot_deg_median": float(np.median(r1)), "rot_deg_max": float(r1.max()),
                                 "centre_m_median": float(np.median(t1e)), "centre_m_max": float(t1e.max())}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
