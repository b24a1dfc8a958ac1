#!/usr/bin/env python
"""bench_fusion.py — RGB-D fusion (AppFusion::fuseSDF on the device: i3d_fusion_begin / integrate / finish) of every rendered depth frame
of a synthetic workload, one JSON line.

    python bench_fusion.py [--workload c3|c2|small|tiny] [--oracle-frames 2]

The workload's depth frames (C3: 200 x 640x480 at 2 mm) and make_color_frames colours are fused with the true poses, one integrate call
per frame, after a two-frame warm-up fusion on the same engine.  Reported: wall ms of the whole fusion (host buffers in, grid installed),
device ms per stage (CUDA events: erosion + normals, allocation, integration, correctSDF, finish), allocated and kept voxels, correctSDF
sweeps, hash growths, and the byte model of k_fuse_integrate (36 B per allocated voxel per frame: coordinates 12, sdf / weight / colour
read 12 and written 12) over its device time, as a share of the HBM peak (MEASURED_PEAKS.json hbm_gbs if present, else the H100 SXM data
sheet's 3350 GB/s).  `oracle_first_frames`: the float CPU restatement (tests/native/fusion_oracle.cpp, single thread) on the first frames
only, labelled as such.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return out.stdout.strip() or None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--oracle-frames", type=int, default=2)
    args = ap.parse_args()

    from fusion_ref import FusionOracle, depth_range, scene_inputs
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene, make_color_frames

    peak_gbs, peak_src = 3350.0, "data sheet 3350 GB/s (H100 SXM HBM3, not measured)"
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peaks = json.load(open(pk))
        if "hbm_gbs" in peaks:
            peak_gbs, peak_src = float(peaks["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"

    import torch
    scene = config_scene(args.workload, device="cuda:0" if torch.cuda.is_available() else "cpu")
    dcam, depth, ccam, _, c2w, w2c = scene_inputs(scene)
    bgr = make_color_frames(scene)
    p = engine.default_fusion_params()
    p.voxel_size = float(scene["voxel_size"])
    p.depth_min, p.depth_max = depth_range(scene)
    F = int(depth.shape[0])

    e = engine.Engine(0)
    e.fusion_begin(p)
    e.fusion_integrate(dcam, depth[:2], ccam, bgr[:2], c2w[:2], w2c[:2])
    e.fusion_finish()

    t0 = time.perf_counter()
    e.fusion_begin(p)
    voxel_frames = 0
    for f in range(F):
        e.fusion_integrate(dcam, depth[f:f + 1], ccam, bgr[f:f + 1], c2w[f:f + 1], w2c[f:f + 1])
        voxel_frames += int(e.L.i3d_debug_fusion_num_voxels(e.h))
    allocated = int(e.L.i3d_debug_fusion_num_voxels(e.h))
    kept = e.fusion_finish()
    wall = time.perf_counter() - t0

    stages = {k: e.phase_ms("fusion_" + k) for k in ("prep", "alloc", "integrate", "correct", "finish")}
    bytes_int = 36.0 * voxel_frames
    gbs = bytes_int / (stages["integrate"] * 1e-3) / 1e9 if stages["integrate"] > 0 else None

    nf = max(0, min(args.oracle_frames, F))
    o = FusionOracle(p.voxel_size, p.depth_min, p.depth_max, p.integration_weight_sample, list(p.clip_bounds), p.discont_window_size,
                     p.correct_sdf_iterations)
    t1 = time.perf_counter()
    o.integrate(dcam, depth[:nf], ccam, bgr[:nf], c2w[:nf], w2c[:nf])
    t_or = time.perf_counter() - t1

    line = {"metric": "fusion_wall_ms", "value": 1e3 * wall, "unit": "ms", "higher_is_better": False, "workload": args.workload, "gpu": gpu_info(),
            "call": "i3d_fusion_begin / i3d_fusion_integrate (one call per frame) / i3d_fusion_finish",
            "frames": F, "depth_size": [int(dcam[0]), int(dcam[1])], "voxel_size": float(p.voxel_size), "device_ms": stages,
            "allocated_voxels": allocated, "kept_voxels": int(kept), "correct_sdf_sweeps": e.phase_count("fusion_sweeps"),
            "hash_growths": e.phase_count("fusion_growths"),
            "integrate_bytes_model": bytes_int, "integrate_gbs": gbs, "integrate_share_of_peak": (gbs / peak_gbs) if gbs else None,
            "peak_gbs": peak_gbs, "peak_source": peak_src,
            "oracle_first_frames": {"frames": nf, "cpu_ms_alloc_integrate": 1e3 * t_or, "note": "CPU oracle, single thread, first frames only"}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
