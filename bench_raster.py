#!/usr/bin/env python
"""bench_raster.py — the rasterizer of the resident mesh (i3d_rasterize_keyframes, i3d_rasterize_views) on the C3 grid, one JSON line.

    python bench_raster.py [--workload c3|c2|small|tiny] [--reps 5] [--quality c2,c3]

Speed: the workload's refined mesh without the component filter, full and simplified at cells of 2, 4 and 8 voxels.  Per mesh, the
median of --reps calls after one warm-up call of: the statistics of every keyframe with vertex colours (planes=(), device ms per stage,
ms per view, (tile, face) pairs and ray-triangle tests per second); all planes of one keyframe (device ms, and wall ms of the call with
the download into numpy); for the full mesh one 1920 x 1080 new view from keyframe 0's pose and one from the centre of the mesh's box,
where faces straddle the camera plane (device ms per stage).  For scale, i3d_render_keyframes' statistics of the same keyframes
(geometry only) in the same run.

Byte and test model, kept here.  k_rast_faces: per (face, view) 12 B of indices and 36 B of vertices, per kept (tile, face) pair a 16 B
tile box, per test an 8 B ray and one 64-bit atomicMin on a hit; it is bound by the tests it runs (latency of the per-pair loop), so it
is reported as tests per second.  k_rast_shade: per pixel an 8 B key and an 8 B ray, for a hit 48 B of face and vertices, 4 B of frame
depth and 3 B of frame colour, plus the planes written (4 + 4 + 8 + 12 + 3 B); it is reported as GB/s of that model against the H100 SXM
data sheet's 3350 GB/s.

Quality (--quality): per scene the texture is baked (12 texels per face, K = 5) from the even keyframes only (their frames, camera and
colour frames uploaded, then bake_texture; the vertex colours are recomputed from the same frames before the extraction), then the odd
keyframes are uploaded and rasterized.  Reported per mesh: mean absolute colour error per channel (R, G, B, uint8 units) of the texture
and of the vertex colours on the held-out odd keyframes, and the same on the even (training) keyframes.  The GPU name and power limit
are read in the same run.  Writes nothing.
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


def shade_bytes(pixels, covered, with_frames):
    return 16 * pixels + (48 + (7 if with_frames else 0)) * covered


def mesh_of(e, vs, cell):
    m = e.extract_mesh("refined", False)
    return e.simplify_mesh(cell * vs) if cell else m


def speed(e, vs, cell, reps, W, H):
    mesh_of(e, vs, cell)
    ids = list(range(e.F))
    e.rasterize_keyframes(ids, "vertex", planes=())
    runs = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = e.rasterize_keyframes(ids, "vertex", planes=())
        runs.append((1e3 * (time.perf_counter() - t0), r["info"]))
    i = runs[0][1]
    med = lambda k: float(np.median([getattr(x[1], k) for x in runs]))
    faces_ms, shade_ms, rays_ms = med("ms_faces"), med("ms_shade"), med("ms_rays")
    dev = rays_ms + faces_ms + shade_ms
    out = {"cell_voxels": cell or 0, "faces": int(i.num_faces), "views": len(ids), "pairs": int(i.num_pairs), "tests": int(i.num_tests),
           "straddling": int(i.num_straddling), "covered": int(i.num_covered), "ms_rays": rays_ms, "ms_faces": faces_ms, "ms_shade": shade_ms,
           "device_ms": dev, "ms_per_view": dev / len(ids), "wall_ms": float(np.median([x[0] for x in runs])),
           "pairs_per_s": int(i.num_pairs) / (faces_ms * 1e-3), "tests_per_s": int(i.num_tests) / (faces_ms * 1e-3)}
    out["shade_gbs"] = shade_bytes(len(ids) * W * H, int(i.num_covered), True) / (shade_ms * 1e-3) / 1e9
    out["shade_share_of_3350"] = out["shade_gbs"] / PEAK_GBS
    # all planes of one keyframe
    e.rasterize_keyframes([0], "vertex")
    devs, walls = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = e.rasterize_keyframes([0], "vertex")
        walls.append(1e3 * (time.perf_counter() - t0))
        devs.append(r["info"].ms_rays + r["info"].ms_faces + r["info"].ms_shade)
    out["one_keyframe_all_planes"] = {"device_ms": float(np.median(devs)), "wall_ms": float(np.median(walls))}
    return out


def new_view(e, vs, reps, inside=False):
    """one 1920 x 1080 view of the full mesh from keyframe 0's pose, or (inside) from the centre of the mesh's box looking along +z"""
    import render_ref as rr
    V = mesh_of(e, vs, None)["vertices"]
    if inside:
        c = (V.min(0) + V.max(0)) / 2
        pose = np.array([[1, 0, 0, 0, 1, 0, 0, 0, 1, -c[0], -c[1], -c[2]]], np.float32)
    else:
        pose = rr.pose_rt(e.download_state()["poses"][:1])
    cam = dict(fx=1500.0, fy=1500.0, cx=959.5, cy=539.5, width=1920, height=1080)
    e.rasterize_views(cam, pose)
    runs = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = e.rasterize_views(cam, pose)
        runs.append((1e3 * (time.perf_counter() - t0), r["info"]))
    med = lambda k: float(np.median([getattr(x[1], k) for x in runs]))
    i = runs[0][1]
    return {"size": [1920, 1080], "inside_the_box": inside, "ms_rays": med("ms_rays"), "ms_faces": med("ms_faces"), "ms_shade": med("ms_shade"),
            "device_ms": med("ms_rays") + med("ms_faces") + med("ms_shade"), "wall_ms": float(np.median([x[0] for x in runs])),
            "covered": int(i.num_covered), "tests": int(i.num_tests), "pairs": int(i.num_pairs), "straddling": int(i.num_straddling)}


def render_scale(e, reps):
    ids = list(range(e.F))
    e.render_keyframes(ids, planes=(), photometric=False)
    ms = []
    for _ in range(reps):
        e.render_keyframes(ids, planes=(), photometric=False)
        ms.append(e.phase_ms("render"))
    return {"views": len(ids), "device_ms": float(np.median(ms))}


def mean_abs(stats):
    n = sum(s["color_count"] for s in stats)
    return [sum(s["color_abs"][k] for s in stats) / max(1, n) for k in range(3)]


def quality(name, device):
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = config_scene(name, device=device)
    col = make_color_frames(s)
    F = len(s["poses"])
    even, odd = np.arange(0, F, 2), np.arange(1, F, 2)
    vs = float(np.float32(s["voxel_size"]))
    e = engine.Engine(0)
    e.load_scene(s)

    def use(sel):
        e.upload_frames(s["lum"][sel], s["depth"][sel], s.get("pyr_scale", 1.0))
        e.set_camera(s["poses"][sel], s["intr"], s["dist"])
        e.upload_color_frames(col[sel])
    rows = []
    for cell in (None, 2, 4, 8):
        use(even)
        e.recompute_colors(0.02, 5)
        mesh_of(e, vs, cell)
        e.bake_texture(12)
        train = {c: mean_abs(e.rasterize_keyframes(list(range(len(even))), c, planes=())["stats"]) for c in ("texture", "vertex")}
        use(odd)
        held = {c: mean_abs(e.rasterize_keyframes(list(range(len(odd))), c, planes=())["stats"]) for c in ("texture", "vertex")}
        rows.append({"cell_voxels": cell or 0, "held_out_texture": held["texture"], "held_out_vertex": held["vertex"],
                     "train_texture": train["texture"], "train_vertex": train["vertex"]})
    e.close()
    return {"scene": name, "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=("c3", "c2", "small", "tiny"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--quality", default="", help="comma-separated scenes for the held-out colour table, e.g. c2,c3")
    args = ap.parse_args()

    import torch
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    sys.path.insert(0, os.path.join(ROOT, "tests"))

    gpu = gpu_info()
    device = "cuda:0" if torch.cuda.is_available() else "cpu"
    scene = config_scene(args.workload, device=device)
    e = engine.Engine(0)
    e.load_scene(scene)
    e.upload_color_frames(make_color_frames(scene))
    reps = max(1, args.reps)
    vs = float(np.float32(scene["voxel_size"]))
    _, H, W = scene["depth"].shape
    runs = [speed(e, vs, cell, reps, W, H) for cell in (None, 2, 4, 8)]
    view = [new_view(e, vs, reps), new_view(e, vs, reps, inside=True)]
    rend = render_scale(e, reps)
    e.close()
    q = [quality(n, device) for n in args.quality.split(",") if n]
    line = {"metric": "raster_keyframe_stats_device_ms", "value": runs[0]["device_ms"], "unit": "ms", "higher_is_better": False,
            "workload": args.workload, "gpu": gpu, "reps": reps, "runs": runs, "new_view": view, "render_keyframes_stats": rend, "quality": q,
            "peak_gbs": PEAK_GBS}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
