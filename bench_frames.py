#!/usr/bin/env python
"""bench_frames.py — keyframe blur scores and the device RGB-D pyramid on a synthetic workload, one JSON line.

    python bench_frames.py [--workload c3|c2|small|tiny] [--reps 5]

The workload's frames (C3: 200 x 640x480) with make_color_frames colours, every 4th frame box-blurred (5x5), are scored with
i3d_keyframe_scores from host buffers, stored with i3d_upload_rgbd_frames (level-0 luminance given, as the refinement passes it), and
installed level by level with i3d_use_rgbd_level.  Reported, each the median of --reps calls after one warm-up call:
  keyframe_scores     wall ms (host buffers in, scores out) and device ms (CUDA events around the kernels), with the byte model of the
                      kernels (3 B read per pixel) over the device time as a share of the HBM peak (MEASURED_PEAKS.json hbm_gbs if present,
                      else the H100 SXM data sheet's 3350 GB/s);
  upload_rgbd_frames  wall ms;
  use_rgbd_level      device ms and wall ms for levels 2, 1 and 0, next to the wall ms of i3d_upload_frames (+ i3d_upload_color_frames at
                      level 0) of the same planes from host buffers, i.e. what a level switch costs without the store.
The device planes are checked byte for byte against tests/frames_ref.py (`bit_exact`).  Writes nothing.
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


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return out.stdout.strip() or None
    except Exception:
        return None


def box_blur(bgr):
    b = bgr.astype(np.float32)
    for ax in (0, 1):
        b = sum(np.roll(b, s, axis=ax) for s in range(-2, 3)) / np.float32(5.0)
    return np.clip(np.rint(b), 0, 255).astype(np.uint8)


def median_ms(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import frames_ref as R
    import torch
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene, make_color_frames

    peak_gbs, peak_src = 3350.0, "data sheet 3350 GB/s (H100 SXM HBM3, not measured)"
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peaks = json.load(open(pk))
        if "hbm_gbs" in peaks:
            peak_gbs, peak_src = float(peaks["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"

    scene = config_scene(args.workload, device="cuda:0" if torch.cuda.is_available() else "cpu")
    lum = np.ascontiguousarray(scene["lum"], np.float32)
    depth = np.ascontiguousarray(scene["depth"], np.float32)
    bgr = make_color_frames(scene)
    bgr[::4] = np.stack([box_blur(f) for f in bgr[::4]])
    F, H, W = lum.shape
    L, D = R.pyramid(bgr, depth, 3, lum=lum)

    e = engine.Engine(0)
    scores = e.keyframe_scores(bgr)
    reps = max(1, args.reps)
    dev = []

    def score():
        e.keyframe_scores(bgr)
        dev.append(e.phase_ms("keyframe_scores"))
    ks_wall = median_ms(score, reps)
    ks_dev = float(np.median(dev))
    ks_bytes = 3.0 * F * W * H
    ks_gbs = ks_bytes / (ks_dev * 1e-3) / 1e9
    ref_scores = R.blur_scores(bgr[:8])
    blurred = np.zeros(F, bool)
    blurred[::4] = True

    up_wall = median_ms(lambda: e.upload_rgbd_frames(bgr, depth, lum), reps)
    levels, exact = {}, True
    for lvl in (2, 1, 0):
        dev = []

        def use():
            e.use_rgbd_level(lvl)
            dev.append(e.phase_ms("frames_level"))
        use_wall = median_ms(use, reps)
        use_dev = float(np.median(dev))
        lg, dg, cg = e.debug_frames(with_color=(lvl == 0))
        exact = exact and lg.tobytes() == L[lvl].tobytes() and dg.tobytes() == D[lvl].tobytes() and (lvl > 0 or cg.tobytes() == bgr.tobytes())

        def host():
            e.upload_frames(L[lvl], D[lvl], 2.0 ** -lvl)
            if lvl == 0:
                e.upload_color_frames(bgr)
        host_wall = median_ms(host, reps)
        mb = (8.0 + (3.0 if lvl == 0 else 0.0)) * F * L[lvl].shape[1] * L[lvl].shape[2] / 1e6
        levels[str(lvl)] = {"size": [int(L[lvl].shape[2]), int(L[lvl].shape[1])], "use_rgbd_level_device_ms": use_dev, "use_rgbd_level_wall_ms": use_wall,
                            "host_upload_wall_ms": host_wall, "host_upload_mb": mb}

    line = {"metric": "keyframe_scores_wall_ms", "value": ks_wall, "unit": "ms", "higher_is_better": False, "workload": args.workload, "gpu": gpu_info(),
            "frames": F, "size": [W, H], "reps": reps,
            "keyframe_scores": {"wall_ms": ks_wall, "device_ms": ks_dev, "bytes_model": ks_bytes, "gbs": ks_gbs, "share_of_peak": ks_gbs / peak_gbs,
                                "max_abs_err_first8_vs_restatement": float(np.nanmax(np.abs(scores[:8] - ref_scores))),
                                "mean_score_blurred": float(np.nanmean(scores[blurred])), "mean_score_sharp": float(np.nanmean(scores[~blurred]))},
            "upload_rgbd_frames_wall_ms": up_wall, "use_rgbd_level": levels, "bit_exact": bool(exact),
            "peak_gbs": peak_gbs, "peak_source": peak_src}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
