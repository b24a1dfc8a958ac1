#!/usr/bin/env python
"""bench_texture.py — the texture bake of the refined mesh (i3d_bake_texture + i3d_download_texture) on the C3 grid, one JSON line.

    python bench_texture.py [--workload c3|c2|small|tiny] [--reps 5]

The workload's refined mesh without the component filter, full and simplified at cells of 2, 4 and 8 voxels, each baked at 8 and 12
texels per face with the default occlusion distance (0.02 m) and K = 5 from the workload's colour frames (scene.make_color_frames) and
the engine's camera.  Each is the median of --reps bakes after one warm-up bake.  Reported per run: faces, atlas size, owned, observed and
fallback texels, observations, the share of (texel, frame) pairs the frame culling skipped, device ms (CUDA events inside the library)
and wall ms of Engine.bake_texture (bake + download into numpy).

Byte model, kept here: a depth tap of 4 B per visited (texel, frame), 12 B per kept observation (its re-probed depth tap and three colour
bytes, rounded up to the 8 B bilinear footprint), 48 B per owned texel for its face (12 B) and three vertex positions (36 B), and 3 B
written per atlas texel.  It is divided by the device time and shown as a share of the H100 SXM data sheet's 3350 GB/s.  The GPU name and
power limit are read in the same run.  Writes nothing.
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
PEAK_GBS = 3350.0


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return out.stdout.strip() or None
    except Exception:
        return None


def model_bytes(info):
    return (4 * int(info.num_texel_frames_visited) + 12 * int(info.num_observations_kept) + 48 * int(info.num_texels_owned)
            + 3 * int(info.atlas_width) * int(info.atlas_height))


def run(e, vs, cell, S, reps):
    e.extract_mesh("refined", False)
    if cell:
        e.simplify_mesh(cell * vs)
    e.bake_texture(S)
    walls, devs, digest = [], [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        t = e.bake_texture(S)
        walls.append(1e3 * (time.perf_counter() - t0))
        devs.append(t["info"].ms_bake)
        d = hash(t["image"].tobytes() + t["uv"].tobytes())
        assert digest is None or d == digest, "bake not run-to-run identical"
        digest = d
    i = t["info"]
    dev = float(np.median(devs))
    gbs = model_bytes(i) / (dev * 1e-3) / 1e9
    return {"cell_voxels": cell or 0, "texels_per_face": S, "faces": int(i.num_faces), "atlas": [int(i.atlas_width), int(i.atlas_height)],
            "texels_owned": int(i.num_texels_owned), "texels_observed": int(i.num_texels_observed), "texels_fallback": int(i.num_texels_fallback),
            "observations": int(i.num_observations), "observations_kept": int(i.num_observations_kept),
            "culled_share": 1.0 - int(i.num_texel_frames_visited) / max(1, int(i.num_texel_frames_total)),
            "device_ms": dev, "wall_ms": float(np.median(walls)), "bytes_model": model_bytes(i), "gbs": gbs, "share_of_3350": gbs / PEAK_GBS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene, make_color_frames

    gpu = gpu_info()
    scene = config_scene(args.workload, device="cuda:0" if torch.cuda.is_available() else "cpu")
    e = engine.Engine(0)
    e.load_scene(scene)
    e.upload_color_frames(make_color_frames(scene))
    reps = max(1, args.reps)
    vs = float(np.float32(scene["voxel_size"]))
    runs = [run(e, vs, cell, S, reps) for cell in (None, 2, 4, 8) for S in (8, 12)]
    head = next(r for r in runs if r["cell_voxels"] == 4 and r["texels_per_face"] == 12)
    line = {"metric": "texture_bake_wall_ms", "value": head["wall_ms"], "unit": "ms", "higher_is_better": False, "workload": args.workload,
            "gpu": gpu, "reps": reps, "runs": runs, "peak_gbs": PEAK_GBS}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
