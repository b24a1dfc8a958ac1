#!/usr/bin/env python
"""bench_odometry.py — dense RGB-D odometry (i3d_fusion_track_and_integrate_sensor) over every frame of a workload, one JSON line.

    python bench_odometry.py [--workload c3|c2|small|tiny] [--reps 3]

The workload's frames go into the sensor store; each rep begins a fusion and runs the loop over all frames from the true pose of frame 0
(anchored), with the default tracking parameters.  Reported, the median over --reps after one warm-up: the call's wall time (phase
"odometry", host clock, ends in a synchronise) in total and per frame, and the device times of the phases odometry_predict,
odometry_icp and the fusion's fusion_prep / fusion_alloc / fusion_integrate.  Beside it, in the same run: i3d_fusion_integrate_sensor
of all frames at the true poses (device time of the fusion phases) and i3d_track_sensor_frames of all frames against the grid fused at
the true poses (phase "track"), from the true poses.  Pose errors of the loop against the true poses.  The GPU name and power limit are
read in the same run.  Writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_track import gpu_info  # noqa: E402

FUSION_PHASES = ("fusion_prep", "fusion_alloc", "fusion_integrate")


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
    true = tr.aa_to_rt(s["poses_true"])

    names = ("odometry", "odometry_predict", "odometry_icp") + FUSION_PHASES
    runs = {k: [] for k in names}
    digest = None
    for rep in range(max(1, args.reps) + 1):
        e.fusion_begin(p)
        out, infos = e.fusion_track_and_integrate_sensor(ids, true[0])
        d = out.tobytes() + repr(infos).encode()
        assert digest is None or d == digest, "odometry not run-to-run identical"
        digest = d
        if rep > 0:
            for k in names:
                runs[k].append(e.phase_ms(k))
    corr = e.phase_count("odometry_correspondences")
    r, t = tr.pose_errors(out, true)

    # beside it: fusion at the true poses, then tracking of every frame against that grid from the true poses
    fuse_ms, track_ms, fuse_wall = [], [], []
    for rep in range(max(1, args.reps) + 1):
        e.fusion_begin(p)
        t0 = time.perf_counter()
        e.fusion_integrate_sensor(ids, c2w, w2c)
        wall = 1e3 * (time.perf_counter() - t0)
        dev = sum(e.phase_ms(k) for k in FUSION_PHASES)
        e.fusion_finish()
        e.track_sensor_frames(ids, true)
        if rep > 0:
            fuse_ms.append(dev); fuse_wall.append(wall); track_ms.append(e.phase_ms("track"))

    med = {k: float(np.median(v)) for k, v in runs.items()}
    line = {"metric": "odometry_all_frames_ms", "value": med["odometry"], "unit": "ms", "higher_is_better": False, "workload": args.workload,
            "gpu": gpu, "reps": len(runs["odometry"]), "frames": int(F), "size": [int(W), int(H)],
            "wall_ms_per_frame": med["odometry"] / F, "device_phases_ms": {k: med[k] for k in names[1:]},
            "device_ms_per_frame": sum(med[k] for k in names[1:]) / F, "correspondences": int(corr),
            "status_counts": {str(k): int(sum(1 for i in infos if i["status"] == k)) for k in range(5)},
            "pose_error": {"rot_deg_median": float(np.median(r)), "rot_deg_max": float(r.max()),
                           "centre_m_median": float(np.median(t)), "centre_m_max": float(t.max())},
            "beside": {"fusion_integrate_sensor_device_ms": float(np.median(fuse_ms)), "fusion_integrate_sensor_wall_ms": float(np.median(fuse_wall)),
                       "track_sensor_frames_device_ms": float(np.median(track_ms)),
                       "sum_per_frame_ms": (float(np.median(fuse_ms)) + float(np.median(track_ms))) / F}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
