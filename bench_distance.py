#!/usr/bin/env python
"""bench_distance.py — the distance between the resident mesh and a reference surface (i3d_surface_distance, DESIGN.md §6u): its speed
and the quality table of the synthetic scene against its analytic surface (scene.truth_mesh), one JSON line per measurement.

    python bench_distance.py [--workloads c2,c3] [--skip-quality]

Speed: the workload's mesh after one lighting estimate and 10 GN iterations (refined sdf, full marching-cubes resolution) against
truth_mesh at L = 2, both directions, after one warm-up call: device ms per stage (CUDA events), point-triangle tests per sample and per
second, and the bytes the query must read at least (every sample's face corners and the target's vertex positions once) over its time.

Quality, at tau = 0.1, 0.25 and 0.5 voxel and max_distance 2 voxels, against truth_mesh unless stated: (1) the sdf0 mesh; (2) the refined
mesh after one lighting estimate and 10 GN iterations with the defaults; (3) that mesh simplified at 2, 4 and 8 voxels, against the
truth and against the full refined mesh; (4) the mesh of every frame fused at the true poses (bench_fusion.py's path).  Writes nothing.
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


def refined_engine(s):
    """the engine of scene s after one lighting estimate and 10 GN iterations with the default parameters"""
    from intrinsic3d_b200 import engine
    e = engine.Engine(0)
    e.load_scene(s)
    lp = engine.default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    e.estimate_lighting(lp)
    p = engine.default_params()
    p.thres_shell = s["thres_shell"]
    for _ in range(10):
        e.gn_iteration(p)
    return e


def fused_engine(s):
    """an engine holding the grid of every depth frame of s fused at the true poses (bench_fusion.py's path)"""
    from fusion_ref import depth_range, scene_inputs
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import make_color_frames
    dcam, depth, ccam, _, c2w, w2c = scene_inputs(s)
    bgr = make_color_frames(s)
    p = engine.default_fusion_params()
    p.voxel_size = float(s["voxel_size"])
    p.depth_min, p.depth_max = depth_range(s)
    e = engine.Engine(0)
    e.fusion_begin(p)
    for f in range(int(depth.shape[0])):
        e.fusion_integrate(dcam, depth[f:f + 1], ccam, bgr[f:f + 1], c2w[f:f + 1], w2c[f:f + 1])
    e.fusion_finish()
    return e


def row(e, label, name, vs, taus, reference):
    r = e.surface_distance(taus, 2 * vs, 2)
    a, c = r["accuracy"], r["completeness"]
    return {"metric": "distance_quality", "workload": name, "row": label, "reference": reference, "faces": int(r["info"].side[0].num_samples // 4),
            "accuracy_mean_vox": a["mean"] / vs, "accuracy_rms_vox": a["rms"] / vs, "accuracy_max_vox": a["max"] / vs,
            "completeness_mean_vox": c["mean"] / vs, "completeness_rms_vox": c["rms"] / vs, "completeness_max_vox": c["max"] / vs,
            "unmatched_area_share": [a["unmatched_area"] / a["area"], c["unmatched_area"] / c["area"]],
            "tau_vox": [t / vs for t in taus], "precision": r["precision"], "recall": r["recall"], "fscore": r["fscore"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3")
    ap.add_argument("--skip-quality", action="store_true")
    args = ap.parse_args()
    import torch
    from intrinsic3d_b200.scene import config_geometry, config_scene, truth_mesh, truth_mesh_error
    gpu = gpu_info()
    for name in args.workloads.split(","):
        s = config_scene(name, device="cuda:0" if torch.cuda.is_available() else "cpu")
        vs = float(s["voxel_size"])
        taus = [0.1 * vs, 0.25 * vs, 0.5 * vs]
        g = config_geometry(name)
        truth = truth_mesh(**g)
        terr = truth_mesh_error(truth, **g)
        e = refined_engine(s)
        refined = e.extract_mesh("refined", False)
        e.upload_reference_mesh(truth)
        # speed: warm-up, then one timed call
        e.surface_distance(taus, 2 * vs, 2)
        t0 = time.perf_counter()
        r = e.surface_distance(taus, 2 * vs, 2)
        wall = time.perf_counter() - t0
        inf = r["info"]
        sides = []
        for d in range(2):
            sd = inf.side[d]
            src_faces, tgt_faces = (len(refined["faces"]), len(truth["faces"])) if d == 0 else (len(truth["faces"]), len(refined["faces"]))
            tgt_verts = len(truth["vertices"]) if d == 0 else len(refined["vertices"])
            tests = int(sd.point_triangle_tests)
            bytes_min = 36.0 * src_faces + 12.0 * tgt_verts + 12.0 * tgt_faces      # corners of the sampled faces, target vertices and faces
            sides.append({"samples": int(sd.num_samples), "target_faces": tgt_faces, "cell_size_m": float(sd.cell_size), "grid": list(sd.grid),
                          "cell_entries": int(sd.num_cell_entries), "ms_grid": sd.ms_grid, "ms_query": sd.ms_query, "ms_reduce": sd.ms_reduce,
                          "tests": tests, "tests_per_sample": tests / max(1, sd.num_samples),
                          "tests_per_s": tests / (sd.ms_query * 1e-3) if sd.ms_query > 0 else None,
                          "min_bytes_over_query_gbs": bytes_min / (sd.ms_query * 1e-3) / 1e9 if sd.ms_query > 0 else None})
        print(json.dumps({"metric": "distance_device_ms", "workload": name, "gpu": gpu, "L": 2, "value": sum(x["ms_grid"] + x["ms_query"] + x["ms_reduce"] for x in sides) + inf.ms_vertices,
                          "unit": "ms", "wall_ms": 1e3 * wall, "resident_faces": len(refined["faces"]), "truth_faces": len(truth["faces"]),
                          "truth_mesh_error_m": terr, "vertices": int(inf.num_vertices), "ms_vertices": inf.ms_vertices,
                          "vertex_tests": int(inf.vertex_point_triangle_tests), "sides": sides}), flush=True)
        if args.skip_quality:
            continue
        rows = [row(e, "2 refined", name, vs, taus, "truth")]
        e.extract_mesh("fused", False)
        rows.append(row(e, "1 sdf0", name, vs, taus, "truth"))
        for cell in (2, 4, 8):
            e.extract_mesh("refined", False)
            e.simplify_mesh(cell * vs)
            rows.append(row(e, f"3 refined simplified {cell} vox", name, vs, taus, "truth"))
            e.upload_reference_mesh(refined)
            rows.append(row(e, f"3 refined simplified {cell} vox", name, vs, taus, "full refined mesh"))
            e.upload_reference_mesh(truth)
        e.close()
        e = fused_engine(s)
        e.extract_mesh("fused", False)
        e.upload_reference_mesh(truth)
        rows.append(row(e, "4 fused at the true poses", name, vs, taus, "truth"))
        e.close()
        for x in rows:
            x["gpu"] = gpu
            print(json.dumps(x), flush=True)


if __name__ == "__main__":
    main()
