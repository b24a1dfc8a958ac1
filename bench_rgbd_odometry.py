#!/usr/bin/env python
"""bench_rgbd_odometry.py — dense RGB-D odometry depth-only (i3d_fusion_track_and_integrate_sensor) and with the photometric term
(i3d_fusion_track_and_integrate_sensor_rgbd) side by side over every frame of a workload, one JSON line.

    python bench_rgbd_odometry.py [--workload c2|c3|small|tiny] [--frames 200] [--weights 0.1] [--ref-weights 0.01,0.05]
                                  [--lni-weights 0.002] [--lni-radius 5] [--lni-eps 0.01] [--clean-color] [--reps 1]

The workload's frames go into the sensor store; each run begins a fusion and runs the loop over all frames from the true pose of frame 0
(anchored) with the default tracking parameters, once depth-only and once per colour weight in --weights (lambda for every level, the
other colour parameters at their defaults).  Reported per mode, the median over --reps after one warm-up of the first mode: status counts,
pose errors against the true poses (median and max), the first frame that breaks the 0.2 deg / 2 mm gates, the wall time (phase "odometry",
host clock, ends in a synchronise) in total and per frame, and the device phases.  For each colour mode one more run with the per-kernel
timers gives the time of k_track_photo_rows ("track_photo_rows") and its byte-model share of 3350 GB/s.  The GPU name and power limit are
read in the same run.  --ref-weights adds, in the same format, one mode per weight of the loop with the reference model
(i3d_fusion_track_and_integrate_sensor_rgbd_ref, DESIGN.md §6q), whose timed run gives k_track_ref_model ("track_ref_model") and its
byte-model share.  --lni-weights adds one mode per weight of the reference loop with locally normalised intensity (norm_radius
--lni-radius, norm_eps --lni-eps, the other colour parameters at i3d_default_track_color_lni_params, DESIGN.md §6r), whose timed run also
gives k_track_local_norm ("track_local_norm") and its byte-model share.  --clean-color stores colour frames with B = G = R =
rint(255 lum) and no per-frame modulation: the bound any appearance compensation can reach with the photometric term.  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_track import gpu_info  # noqa: E402

PHASES = ("odometry_predict", "odometry_icp", "fusion_prep", "fusion_alloc", "fusion_integrate")
HBM_GBS = 3350.0
# k_track_photo_rows' byte model per pixel of a level and per system, an upper bound as if every pixel passed every gate: prediction
# depth and model intensity (8 B), the occlusion depth tap (4 B), four bilinear taps of intensity, grad_x and grad_y (48 B)
PHOTO_BYTES_PER_PIXEL = 60
# k_track_ref_model's byte model per pixel of a level and per frame, an upper bound as if every pixel passed every test: prediction depth
# (4 B), the reference depth tap (4 B), four intensity taps (16 B) and the model write (4 B)
REF_BYTES_PER_PIXEL = 28
# k_track_local_norm's byte model per pixel of a level: one read of the raw plane and one write of the normalised plane (8 B); the halo
# rows and the (2r+1) taps along the row and down the column come from L1 / shared memory
LNI_BYTES_PER_PIXEL = 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--weights", default="0.1")
    ap.add_argument("--ref-weights", default="")
    ap.add_argument("--lni-weights", default="")
    ap.add_argument("--lni-radius", type=int, default=5)
    ap.add_argument("--lni-eps", type=float, default=0.01)
    ap.add_argument("--clean-color", action="store_true")
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()

    import torch
    import track_ref as tr
    from fusion_ref import depth_range, scene_inputs
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene

    gpu = gpu_info()
    s = config_scene(args.workload, device="cuda:0" if torch.cuda.is_available() else "cpu", frames=args.frames)
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    F, H, W = depth.shape
    if args.clean_color:
        bgr = np.repeat(np.clip(np.rint(np.asarray(s["lum"], np.float32) * np.float32(255.0)), 0, 255).astype(np.uint8)[..., None], 3, axis=-1)
    e = engine.Engine(0)
    e.sensor_frames_begin(dcam, ccam, F)
    e.sensor_frames_add(depth, bgr)
    p = engine.default_fusion_params()
    p.voxel_size = float(s["voxel_size"])
    p.depth_min, p.depth_max = depth_range(s)
    ids = np.arange(F, dtype=np.int32)
    true = tr.aa_to_rt(s["poses_true"])
    tp = engine.default_track_params()
    pixels_per_frame = sum(tp.iterations[l] * (W >> l) * (H >> l) for l in range(tp.num_levels))
    level_pixels = sum((W >> l) * (H >> l) for l in range(tp.num_levels))

    def run(mode, timers=False):
        e.set_kernel_timers(1 if timers else 0)
        e.fusion_begin(p)
        ref, weight = mode
        if weight is None:
            out, infos = e.fusion_track_and_integrate_sensor(ids, true[0])
        elif ref == "lni":
            out, infos = e.fusion_track_and_integrate_sensor_rgbd_ref(ids, true[0], color=dict(weight=weight, norm_radius=args.lni_radius,
                                                                                                norm_eps=args.lni_eps))
        elif ref:
            out, infos = e.fusion_track_and_integrate_sensor_rgbd_ref(ids, true[0], color=dict(weight=weight))
        else:
            out, infos = e.fusion_track_and_integrate_sensor_rgbd(ids, true[0], color=dict(weight=weight))
        e.set_kernel_timers(0)
        return out, infos

    modes = [(False, None)] + [(False, float(w)) for w in args.weights.split(",")]
    modes += [(True, float(w)) for w in args.ref_weights.split(",") if w]
    modes += [("lni", float(w)) for w in args.lni_weights.split(",") if w]
    run(modes[0])                                                       # warm-up
    results = {}
    for mode in modes:
        ref, w = mode
        wall, dev = [], {k: [] for k in PHASES}
        for _ in range(max(1, args.reps)):
            out, infos = run(mode)
            wall.append(e.phase_ms("odometry"))
            for k in PHASES:
                dev[k].append(e.phase_ms(k))
        r, t = tr.pose_errors(out, true)
        st = [i["status"] for i in infos]
        bad = [k for k in range(F) if st[k] not in (0, 4) or r[k] > 0.2 or t[k] > 0.002]
        res = {"status_counts": {str(k): int(sum(1 for x in st if x == k)) for k in range(5)},
               "pose_error": {"rot_deg_median": float(np.median(r)), "rot_deg_max": float(r.max()),
                              "centre_m_median": float(np.median(t)), "centre_m_max": float(t.max())},
               "first_frame_over_gates": bad[0] if bad else None,
               "wall_ms": float(np.median(wall)), "wall_ms_per_frame": float(np.median(wall)) / F,
               "device_phases_ms": {k: float(np.median(v)) for k, v in dev.items()},
               "device_ms_per_frame": sum(float(np.median(v)) for v in dev.values()) / F,
               "correspondences": int(e.phase_count("odometry_correspondences"))}
        if w is not None:
            res["photo_correspondences"] = int(e.phase_count("odometry_photo_correspondences"))
            run(mode, timers=True)
            ms = e.phase_ms("track_photo_rows")
            gb = F * pixels_per_frame * PHOTO_BYTES_PER_PIXEL / 1e9
            res["k_track_photo_rows"] = {"ms": ms, "launches": int(e.phase_count("track_photo_rows")), "model_gb": gb,
                                         "gbs": gb / (ms / 1e3) if ms > 0 else None,
                                         "share_of_hbm": gb / (ms / 1e3) / HBM_GBS if ms > 0 else None}
            if ref:
                ms = e.phase_ms("track_ref_model")
                n = int(e.phase_count("track_ref_model"))
                gb = n // tp.num_levels * level_pixels * REF_BYTES_PER_PIXEL / 1e9
                res["k_track_ref_model"] = {"ms": ms, "launches": n, "model_gb": gb, "gbs": gb / (ms / 1e3) if ms > 0 else None,
                                            "share_of_hbm": gb / (ms / 1e3) / HBM_GBS if ms > 0 else None}
            if ref == "lni":
                ms = e.phase_ms("track_local_norm")
                n = int(e.phase_count("track_local_norm"))
                gb = n // tp.num_levels * level_pixels * LNI_BYTES_PER_PIXEL / 1e9
                res["k_track_local_norm"] = {"ms": ms, "launches": n, "ms_per_frame": ms / F, "model_gb": gb,
                                             "gbs": gb / (ms / 1e3) if ms > 0 else None,
                                             "share_of_hbm": gb / (ms / 1e3) / HBM_GBS if ms > 0 else None}
        if w is None:
            key = "depth_only"
        elif ref == "lni":
            key = f"lni_r{args.lni_radius}_eps{args.lni_eps:g}_w{w:g}"
        else:
            key = f"ref_w{w:g}" if ref else f"color_w{w:g}"
        results[key] = res
    line = {"metric": "rgbd_odometry_all_frames_ms", "value": results[f"color_w{modes[1][1]:g}"]["wall_ms"], "unit": "ms",
            "higher_is_better": False, "workload": args.workload, "gpu": gpu, "reps": max(1, args.reps), "frames": int(F),
            "size": [int(W), int(H)], "clean_color": bool(args.clean_color), "modes": results}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
