#!/usr/bin/env python
"""bench_mesh.py — surface extraction (i3d_extract_mesh + i3d_download_mesh) on the C3 grid and on its 8x upsample, one JSON line.

    python bench_mesh.py [--workload c3|c2|small|tiny] [--reps 5]

Runs, each the median of --reps calls after one warm-up call: both sdf sources with and without the component filter on the workload's
grid (C3: 2 M voxels), then the refined source with and without the filter on the grid after one i3d_upsample_grid (C3: 16 M voxels).
On both grids, after a lighting estimate, the refined mesh coloured by the "albedo" and "shading_sv" modes, with the device time of the
colour pass (phase "mesh_colorize") beside the stage times, its share of the extraction's device time and its byte model.
Reported per run: the counts of every stage, device ms per stage (CUDA events inside the library), wall ms of Engine.extract_mesh
(extraction + download into numpy), and the byte models of the two per-voxel kernels over their device time as a share of the HBM peak
(MEASURED_PEAKS.json hbm_gbs if present, else the H100 SXM data sheet's 3350 GB/s):
  classify  per voxel: 7 neighbour ids (28 B), coordinates (12 B), weight (4 B), sdf (8 B) read, case (1 B) and count (4 B) written,
            plus the 16 B of the offset scan (the corner loads of other voxels are assumed to hit the cache);
  emit      per voxel the count (4 B); per triangle corner position (12 B), colour (3 B) and sort keys (12 B) written.
The GPU name and power limit are read in the same run.  Writes nothing.
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

STAGES = ("ms_classify", "ms_emit", "ms_weld", "ms_clean", "ms_components")
# bytes per voxel of the colour pass: albedo reads the albedo (8 B) and writes a colour (4 B); shading_sv reads the weights of the voxel
# and its +x/+y/+z neighbours (16 B), the 3 neighbour slots (12 B), 4 sdf values (32 B), the albedo (8 B) and the coordinates (12 B) and
# writes 4 B (the subvolume SH, a few kB, stay in cache)
COLORIZE_BYTES = {"albedo": 12, "shading_sv": 84}
COUNTS = ("num_cubes", "num_faces_raw", "num_vertices_welded", "num_faces_clean", "num_faces", "num_vertices")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return out.stdout.strip() or None
    except Exception:
        return None


def run(e, source, lc, reps, peak_gbs, mode=""):
    e.extract_mesh(source, lc, mode)
    walls, infos, colorize, digest = [], [], [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        m = e.extract_mesh(source, lc, mode)
        walls.append(1e3 * (time.perf_counter() - t0))
        infos.append(m["info"])
        colorize.append(e.phase_ms("mesh_colorize") if mode else 0.0)
        d = hash(m["vertices"].tobytes() + m["colors"].tobytes() + m["faces"].tobytes())
        assert digest is None or d == digest, "extraction not run-to-run identical"
        digest = d
    info = infos[0]
    dev = {k: float(np.median([getattr(i, k) for i in infos])) for k in STAGES}
    n, M = e.n, 3 * int(info.num_faces_raw)
    cls_bytes, emit_bytes = n * (28 + 12 + 4 + 8 + 1 + 4 + 16), n * 4 + M * 27
    cls_gbs = cls_bytes / (dev["ms_classify"] * 1e-3) / 1e9
    emit_gbs = emit_bytes / (dev["ms_emit"] * 1e-3) / 1e9 if dev["ms_emit"] > 0 else 0.0
    out = {"source": source, "largest_component_only": bool(lc), "color_mode": mode, "voxels": int(n), **{k: int(getattr(info, k)) for k in COUNTS},
           "device_ms": {**dev, "total": float(sum(dev.values()))}, "wall_ms": float(np.median(walls)),
            "classify": {"bytes_model": cls_bytes, "gbs": cls_gbs, "share_of_peak": cls_gbs / peak_gbs},
            "emit": {"bytes_model": emit_bytes, "gbs": emit_gbs, "share_of_peak": emit_gbs / peak_gbs}}
    if mode:
        col_ms = float(np.median(colorize))
        col_bytes = n * COLORIZE_BYTES[mode]
        col_gbs = col_bytes / (col_ms * 1e-3) / 1e9
        out["colorize"] = {"device_ms": col_ms, "share_of_extraction": col_ms / out["device_ms"]["total"], "bytes_model": col_bytes,
                           "gbs": col_gbs, "share_of_peak": col_gbs / peak_gbs}
    return out


def light(e, scene):
    """a lighting estimate of the current grid (0.2 m subvolumes, as data/intrinsic3d.yml), which the shading modes blend"""
    from intrinsic3d_b200 import engine
    lp = engine.default_lighting_params()
    lp.thres_shell = scene["thres_shell"]
    lp.subvolume_size = 0.2
    e.estimate_lighting(lp)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene

    peak_gbs, peak_src = 3350.0, "data sheet 3350 GB/s (H100 SXM HBM3, not measured)"
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peaks = json.load(open(pk))
        if "hbm_gbs" in peaks:
            peak_gbs, peak_src = float(peaks["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    gpu = gpu_info()
    scene = config_scene(args.workload, device="cuda:0" if torch.cuda.is_available() else "cpu")
    e = engine.Engine(0)
    e.load_scene(scene)
    reps = max(1, args.reps)
    runs = [run(e, src, lc, reps, peak_gbs) for src in ("fused", "refined") for lc in (False, True)]
    light(e, scene)
    runs += [run(e, "refined", False, reps, peak_gbs, mode) for mode in ("albedo", "shading_sv")]
    e.upsample_grid()
    runs += [run(e, "refined", lc, reps, peak_gbs) for lc in (False, True)]
    light(e, scene)
    runs += [run(e, "refined", False, reps, peak_gbs, mode) for mode in ("albedo", "shading_sv")]
    line = {"metric": "mesh_refined_wall_ms", "value": runs[2]["wall_ms"], "unit": "ms", "higher_is_better": False, "workload": args.workload,
            "gpu": gpu, "reps": reps, "runs": runs, "peak_gbs": peak_gbs, "peak_source": peak_src}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
