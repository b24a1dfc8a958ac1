#!/usr/bin/env python
"""bench_mesh_simplify.py — mesh simplification by quadric-error vertex clustering (i3d_simplify_mesh + i3d_download_mesh) on the C3 grid
and on its 8x upsample, one JSON line.

    python bench_mesh_simplify.py [--workload c3|c2|small|tiny] [--reps 5]

On the workload's grid (C3: 2 M voxels) and after one i3d_upsample_grid (C3: 16 M voxels): the refined mesh without the component
filter, simplified at cell sizes of 2, 4 and 8 voxels (of that grid).  Each is the median of --reps calls after one warm-up call; every
call simplifies a fresh extraction (the extraction is not timed with it).  Reported per run: faces and vertices in and out, the counts
of the simplification, device ms per stage (CUDA events inside the library), wall ms of Engine.simplify_mesh (simplification + download
into numpy) beside the wall ms of Engine.extract_mesh on the same grid, and per stage a byte model over its device time as a share of
the HBM peak (MEASURED_PEAKS.json hbm_gbs if present, else the H100 SXM data sheet's 3350 GB/s).

Byte model: what each kernel and CUB pass has to read and write once; a radix sort counts as one read and one write of its keys and
values, although CUB makes several digit passes, and an array gathered at random (positions, quadrics) counts once per element, as if
every repeat hit the cache.
  cluster         per input vertex 156 B: position (12 B) read, cell keys (12 B) written, the two sorts (16 B, 24 B), the gather of the
                  x|y keys (20 B), the segment heads (36 B), the two scans (16 B) and the cluster ids (20 B)
  quadrics        per input face 84 B: the face (12 B), the quadric (72 B); per input vertex its position (12 B)
  representatives per corner (3 per input face) 40 B: corner keys (16 B), their sort (16 B), the runs (4 B), the corner id (4 B); per
                  input face its quadric (72 B); per input vertex 23 B (sorted id, segment head, position, colour); per cluster 27 B
  faces           per input face 191 B: the face and its cluster ids (24 B), cluster face and keys (24 B), iota (4 B), the two sorts
                  (16 B, 24 B), the gather (20 B), k_face_clean (13 B), the duplicate test (41 B), the select (25 B); per cluster its
                  representative (12 B)
  compact         per cluster 50 B (mark, scan, move of 15 B); per output face 36 B (mark, renumber)
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

STAGES = ("ms_cluster", "ms_quadrics", "ms_representatives", "ms_faces", "ms_compact")
COUNTS = ("num_clusters", "num_faces_collapsed", "num_faces_duplicate", "num_faces_degenerate", "num_faces", "num_vertices")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return out.stdout.strip() or None
    except Exception:
        return None


def stage_bytes(V, F, K, F2):
    return {"ms_cluster": 156 * V, "ms_quadrics": 84 * F + 12 * V, "ms_representatives": 40 * 3 * F + 72 * F + 23 * V + 27 * K,
            "ms_faces": 191 * F + 12 * K, "ms_compact": 50 * K + 36 * F2}


def extract_wall(e, reps):
    e.extract_mesh("refined", False)
    walls = []
    for _ in range(reps):
        t0 = time.perf_counter()
        m = e.extract_mesh("refined", False)
        walls.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(walls)), m


def run(e, voxel_size, factor, reps, peak_gbs, extract_ms, m_in):
    cell = factor * voxel_size
    e.extract_mesh("refined", False)
    e.simplify_mesh(cell)
    walls, infos, digest = [], [], None
    for _ in range(reps):
        e.extract_mesh("refined", False)
        t0 = time.perf_counter()
        s = e.simplify_mesh(cell)
        walls.append(1e3 * (time.perf_counter() - t0))
        infos.append(s["info"])
        d = hash(s["vertices"].tobytes() + s["colors"].tobytes() + s["faces"].tobytes())
        assert digest is None or d == digest, "simplification not run-to-run identical"
        digest = d
    info = infos[0]
    dev = {k: float(np.median([getattr(i, k) for i in infos])) for k in STAGES}
    V, F = len(m_in["vertices"]), len(m_in["faces"])
    model = stage_bytes(V, F, int(info.num_clusters), int(info.num_faces))
    bw = {}
    for k in STAGES:
        gbs = model[k] / (dev[k] * 1e-3) / 1e9 if dev[k] > 0 else 0.0
        bw[k] = {"bytes_model": model[k], "gbs": gbs, "share_of_peak": gbs / peak_gbs}
    return {"voxels": int(e.n), "cell_voxels": factor, "cell_size": cell, "faces_in": F, "vertices_in": V, **{k: int(getattr(info, k)) for k in COUNTS},
            "face_ratio": int(info.num_faces) / F, "device_ms": {**dev, "total": float(sum(dev.values()))}, "bandwidth": bw,
            "wall_ms": float(np.median(walls)), "extract_wall_ms": extract_ms}


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
    vs = float(np.float32(scene["voxel_size"]))
    runs = []
    for level in range(2):
        ex_ms, m = extract_wall(e, reps)
        runs += [run(e, vs, f, reps, peak_gbs, ex_ms, m) for f in (2, 4, 8)]
        if level == 0:
            e.upsample_grid()
            vs /= 2
    line = {"metric": "mesh_simplify_wall_ms", "value": runs[1]["wall_ms"], "unit": "ms", "higher_is_better": False, "workload": args.workload,
            "gpu": gpu, "reps": reps, "runs": runs, "peak_gbs": peak_gbs, "peak_source": peak_src}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
