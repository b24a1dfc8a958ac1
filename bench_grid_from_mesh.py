#!/usr/bin/env python
"""bench_grid_from_mesh.py — the voxel grid from a triangle mesh (i3d_grid_from_mesh, DESIGN.md §6v): its speed and the per-voxel
table of the synthetic scene against the converted truth mesh, one JSON line per measurement.

    python bench_grid_from_mesh.py [--workloads c2,c3] [--skip-quality]

Speed: the workload's truth_mesh, and its refined mesh after one lighting estimate and 10 GN iterations (bench_distance.py's schedule),
converted at the scene's voxel size and band 3 after one warm-up call: device ms per stage (CUDA events), candidate and emitted voxels,
point-triangle tests per second of the query stage.

Quality: the truth mesh converted on the scene's lattice is an exact signed-distance grid (to the tessellation's error); on the voxels
both grids hold, the median, p95 and max of |sdf0 - truth| and |sdf_refined - truth| in voxels.  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_distance import gpu_info, refined_engine  # noqa: E402


def convert(e, vs, source, remesh=None):
    """one warm-up call, then the timed one; remesh re-extracts the resident mesh a conversion replaced"""
    e.grid_from_mesh(source, vs, 3.0)
    if remesh:
        remesh()
    n, info = e.grid_from_mesh(source, vs, 3.0)
    d = info.as_dict()
    d["tests_per_s"] = info.point_triangle_tests / (info.ms_query * 1e-3) if info.ms_query > 0 else None
    return n, d


def per_voxel(xyz, values, txyz, tsdf, vs):
    key = lambda a: a.astype(np.int64) @ np.array([1 << 42, 1 << 21, 1], np.int64)   # noqa: E731
    ka, kt = key(xyz + (1 << 20)), key(txyz + (1 << 20))
    common, ia, it = np.intersect1d(ka, kt, assume_unique=True, return_indices=True)
    out = {"voxels_shared": int(len(common))}
    for name, v in values.items():
        d = np.abs(v[ia] - tsdf[it]) / vs
        out[name] = dict(median=float(np.median(d)), p95=float(np.percentile(d, 95)), max=float(d.max()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3")
    ap.add_argument("--skip-quality", action="store_true")
    a = ap.parse_args()
    import torch
    from intrinsic3d_b200.scene import config_geometry, config_scene, truth_mesh
    gpu = gpu_info()
    for name in a.workloads.split(","):
        s = config_scene(name, device="cuda" if torch.cuda.is_available() else "cpu")
        vs = float(s["voxel_size"])
        truth = truth_mesh(None, **config_geometry(name))
        e = refined_engine(s)
        g = e.download_grid()
        refined = e.extract_mesh("refined", False)

        def remesh():
            e.upload_grid(g["xyz"], g["sdf0"], g["sdf_refined"], g["albedo"], g["weight"], g["rgb"], vs)
            e.extract_mesh("refined", False)
        n, info = convert(e, vs, "resident", remesh)
        print(json.dumps(dict(bench="grid_from_mesh", workload=name, mesh="refined", faces=len(refined["faces"]), voxels=n, gpu=gpu, **info)))
        e.upload_reference_mesh(truth)
        n, info = convert(e, vs, "reference")
        print(json.dumps(dict(bench="grid_from_mesh", workload=name, mesh="truth", faces=len(truth["faces"]), voxels=n, gpu=gpu, **info)))
        if not a.skip_quality:
            t = e.download_grid()
            q = per_voxel(g["xyz"], {"sdf0": g["sdf0"], "sdf_refined": g["sdf_refined"]}, t["xyz"], t["sdf0"], vs)
            print(json.dumps(dict(bench="grid_from_mesh_quality", workload=name, gpu=gpu, **q)))
        e.close()


if __name__ == "__main__":
    main()
