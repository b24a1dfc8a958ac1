#!/usr/bin/env python
"""bench_sensor.py — the sensor store (DESIGN.md §6l) against host buffers on a synthetic sequence, one JSON line per workload.

    python bench_sensor.py [--workload c3|c2|small|tiny] [--reps 5] [--only copy|resize]

The workload's depth frames (C3: 200 x 640x480 at 2 mm) and make_color_frames colours run as two workloads:
  copy    colour 640x480 = the depth camera: i3d_select_rgbd_frames copies the depth planes;
  resize  colour 1280x960 (each colour pixel repeated 2x2, a camera with twice the focal length whose pixel centres map onto the depth
          camera's): i3d_select_rgbd_frames runs k_resize_depth.
Reported for each, the median of --reps calls after one warm-up call:
  sensor_upload    wall ms of i3d_sensor_frames_begin + one i3d_sensor_frames_add of every frame;
  keyframe_scores  i3d_sensor_keyframe_scores device ms and wall ms, against i3d_keyframe_scores from host buffers (wall and device ms);
  fusion           i3d_fusion_begin / i3d_fusion_integrate_sensor (all frames) / i3d_fusion_finish wall ms, against one host
                   i3d_fusion_integrate call per frame as bench_fusion.py makes them; the two grids are asserted byte-identical;
  select           i3d_select_rgbd_frames (every frame) + i3d_use_rgbd_level(0) wall ms, against i3d_upload_rgbd_frames of the same planes
                   from host buffers + i3d_use_rgbd_level(0);
  resize_depth     k_resize_depth device ms (resize workload) against its byte model, 4 B read + 4 B written per output pixel, as a share
                   of the HBM peak (MEASURED_PEAKS.json hbm_gbs if present, else the H100 SXM data sheet's 3350 GB/s).
The card's name and power limit are read in the same run.  The selected depth of the first frames is checked byte for byte against
tests/sensor_ref.py.  Writes nothing.
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


def median_ms(fn, reps, dev=None, phase=None, eng=None):
    """Median wall ms of fn() over reps calls after one warm-up; with `phase`, the median device ms of that phase goes to dev[0]."""
    fn()
    t, d = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(1e3 * (time.perf_counter() - t0))
        if phase:
            d.append(eng.phase_ms(phase))
    if phase:
        dev.append(float(np.median(d)))
    return float(np.median(t))


def grid_bytes(e):
    g = e.download_grid()
    return b"".join(np.asarray(g[k]).tobytes() for k in ("xyz", "sdf0", "sdf_refined", "albedo", "weight", "rgb", "voxel_size"))


def run(name, scene, reps, peak_gbs):
    import sensor_ref
    from fusion_ref import depth_range, scene_inputs
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import make_color_frames

    dcam, depth, _, _, c2w, w2c = scene_inputs(scene)
    bgr = make_color_frames(scene)
    W, H, fx, fy, cx, cy = dcam
    if name == "resize":
        ccam = (2 * W, 2 * H, 2 * fx, 2 * fy, 2 * cx + 0.5, 2 * cy + 0.5)
        bgr = np.ascontiguousarray(np.repeat(np.repeat(bgr, 2, axis=1), 2, axis=2))
    else:
        ccam = dcam
    F = int(depth.shape[0])
    ids = np.arange(F, dtype=np.int32)
    p = engine.default_fusion_params()
    p.voxel_size = float(scene["voxel_size"])
    p.depth_min, p.depth_max = depth_range(scene)

    e = engine.Engine(0)

    def upload():
        e.sensor_frames_begin(dcam, ccam, F)
        e.sensor_frames_add(depth, bgr)
    up_wall = median_ms(upload, reps)

    dev = []
    sc_wall = median_ms(lambda: e.sensor_keyframe_scores(), reps, dev, "keyframe_scores", e)
    host_sc_wall = median_ms(lambda: e.keyframe_scores(bgr), reps, dev, "keyframe_scores", e)
    scores_equal = e.sensor_keyframe_scores().tobytes() == e.keyframe_scores(bgr).tobytes()

    def fuse_store():
        e.fusion_begin(p)
        e.fusion_integrate_sensor(ids, c2w, w2c)
        e.fusion_finish()

    def fuse_host():
        e.fusion_begin(p)
        for f in range(F):
            e.fusion_integrate(dcam, depth[f:f + 1], ccam, bgr[f:f + 1], c2w[f:f + 1], w2c[f:f + 1])
        e.fusion_finish()
    fu_store = median_ms(fuse_store, reps)
    g_store = grid_bytes(e)
    fu_host = median_ms(fuse_host, reps)
    assert grid_bytes(e) == g_store, "the store fusion and the host fusion gave different grids"

    def select():
        e.select_rgbd_frames(ids)
        e.use_rgbd_level(0)
    sel_wall = median_ms(select, reps, dev, "resize_depth" if name == "resize" else None, e)
    resize_ms = dev[-1] if name == "resize" else None
    lum0, dep0, bgr0 = e.debug_frames(with_color=True)
    nchk = min(F, 4)
    exact = dep0[:nchk].tobytes() == sensor_ref.resize_depth(depth[:nchk], dcam, ccam).tobytes() and bgr0.tobytes() == bgr.tobytes()

    def host_select():
        e.upload_rgbd_frames(bgr0, dep0)
        e.use_rgbd_level(0)
    host_sel_wall = median_ms(host_select, reps)

    out = {"workload": name, "frames": F, "depth_size": [int(W), int(H)], "color_size": [int(ccam[0]), int(ccam[1])], "reps": reps,
           "sensor_upload_wall_ms": up_wall,
           "keyframe_scores": {"store_device_ms": dev[0], "store_wall_ms": sc_wall, "host_device_ms": dev[1], "host_wall_ms": host_sc_wall,
                               "byte_equal": bool(scores_equal)},
           "fusion": {"store_wall_ms": fu_store, "host_per_frame_wall_ms": fu_host, "grids_byte_identical": True},
           "select": {"select_use_level0_wall_ms": sel_wall, "host_upload_use_level0_wall_ms": host_sel_wall, "first_frames_bit_exact": bool(exact)}}
    if resize_ms is not None:
        model = 8.0 * F * ccam[0] * ccam[1]
        gbs = model / (resize_ms * 1e-3) / 1e9
        out["resize_depth"] = {"device_ms": resize_ms, "bytes_model": model, "gbs": gbs, "share_of_peak": gbs / peak_gbs}
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", choices=("copy", "resize"), default=None)
    args = ap.parse_args()

    import torch
    from intrinsic3d_b200.scene import config_scene

    peak_gbs, peak_src = 3350.0, "data sheet 3350 GB/s (H100 SXM HBM3, not measured)"
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peaks = json.load(open(pk))
        if "hbm_gbs" in peaks:
            peak_gbs, peak_src = float(peaks["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    scene = config_scene(args.workload, device="cuda:0" if torch.cuda.is_available() else "cpu")
    gpu = gpu_info()
    for name in ([args.only] if args.only else ["copy", "resize"]):
        r = run(name, scene, max(1, args.reps), peak_gbs)
        line = {"metric": "sensor_upload_wall_ms", "value": r["sensor_upload_wall_ms"], "unit": "ms", "higher_is_better": False,
                "scene": args.workload, "gpu": gpu, **r, "peak_gbs": peak_gbs, "peak_source": peak_src}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
