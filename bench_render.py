#!/usr/bin/env python
"""bench_render.py — rendering the refined surface into the keyframes (i3d_render_keyframes) on the C3 grid, one JSON line.

    python bench_render.py [--workload c3|c2|small|tiny] [--reps 5]

Runs, each the median of --reps calls after one warm-up call, with empty-space skipping on and off:
  stats_all   statistics only (no planes) for every keyframe of the workload (C3: 200 at 640 x 480);
  planes_one  all five planes for keyframe 0.
Reported per run: device ms of the call (phase "render", CUDA events inside the library) and per view, lattice samples evaluated
(phase count "render_samples") and samples per second, wall ms of Engine.render_keyframes.  The device time of scoring every keyframe is
also given as a share of the 164 ms a C3 refinement level takes (DESIGN.md §5, e2e.refine_level_call on one H100 SXM at 400 W), and the
first render's bitmap build (phase "render_bricks") is reported on its own.  The GPU name and power limit are read in the same run.
Writes nothing.
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

REFINE_LEVEL_MS = 164.0


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return out.stdout.strip() or None
    except Exception:
        return None


def run(e, ids, planes, skip, reps):
    e.set_render_skip(skip)
    e.render_keyframes(ids, planes=planes)
    dev, walls, samples, digest = [], [], [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = e.render_keyframes(ids, planes=planes)
        walls.append(1e3 * (time.perf_counter() - t0))
        dev.append(e.phase_ms("render"))
        samples.append(e.phase_count("render_samples"))
        d = hash(repr(out["stats"]) + "".join(str(hash(out[p].tobytes())) for p in planes))
        assert digest is None or d == digest, "render not run-to-run identical"
        digest = d
    ms = float(np.median(dev))
    st = out["stats"]
    return {"views": len(ids), "planes": list(planes), "skip": skip, "device_ms": ms, "device_ms_per_view": ms / len(ids),
            "wall_ms": float(np.median(walls)), "samples": int(samples[0]), "samples_per_s": samples[0] / (ms * 1e-3),
            "num_hit": int(sum(s["num_hit"] for s in st)),
            "mean_abs_depth_err_m": sum(s["depth_abs"] for s in st) / max(1, sum(s["depth_count"] for s in st)),
            "mean_abs_photo_err": sum(s["photo_abs"] for s in st) / max(1, sum(s["photo_count"] for s in st))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene

    gpu = gpu_info()
    scene = config_scene(args.workload, device="cuda:0" if torch.cuda.is_available() else "cpu")
    e = engine.Engine(0)
    e.load_scene(scene)
    e.render_keyframes([0], planes=())
    bricks_ms = e.phase_ms("render_bricks")
    reps = max(1, args.reps)
    F = scene["depth"].shape[0]
    runs = {}
    for skip in (True, False):
        tag = "skip" if skip else "dense"
        runs["stats_all_" + tag] = run(e, list(range(F)), (), skip, reps)
        runs["planes_one_" + tag] = run(e, [0], ("depth", "normal", "albedo", "shading", "intensity"), skip, reps)
    assert runs["stats_all_skip"]["num_hit"] == runs["stats_all_dense"]["num_hit"]
    score = runs["stats_all_skip"]["device_ms"]
    line = {"metric": "render_stats_all_keyframes_ms", "value": score, "unit": "ms", "higher_is_better": False, "workload": args.workload,
            "gpu": gpu, "reps": reps, "voxels": int(e.n), "keyframes": int(F), "render_bricks_ms": bricks_ms,
            "share_of_refine_level": score / REFINE_LEVEL_MS, "runs": runs}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
