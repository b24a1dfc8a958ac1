#!/usr/bin/env python
"""bench_register.py — registering the reference mesh to the resident mesh (i3d_register_reference_mesh, DESIGN.md §6aa): its speed, its
basin and the surface-distance quality table after registration, one JSON line per measurement, each with the card's name and power limit.

    python bench_register.py [--workloads c2,c3] [--basin tiny,c2,c3] [--skip-quality]

Speed: the sdf0 mesh (fused source, full marching-cubes resolution) against truth_mesh at L = 1 with the default schedule, after one
warm-up call: device ms per iteration split into rows and solve, grid build and total, point-triangle tests per sample and per second, and
whether two calls give the same bytes.

Basin: a copy of the sdf0 mesh moved by a rotation of 0.5, 1, 2, 5 and 10 degrees about its centre (8 seeded axes each) and a translation
of 1, 2 and 4 voxels, registered back with the defaults.  A run converges when T is within 0.001 voxel (largest vertex displacement) and
0.001 degree of the truth.

Quality: i3d_surface_distance at tau = 0.1, 0.25 and 0.5 voxel (max_distance 2 voxels, L = 2) against truth_mesh before and after
registering the truth to (1) the sdf0 mesh, (2) the refined mesh after one lighting estimate and 10 GN iterations, (3) the mesh fused from
the first 25 frames by dense odometry; with the recovered rotation (degrees) and translation (voxels).  Writes nothing.
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_distance import gpu_info, refined_engine  # noqa: E402

ROTATIONS = (0.5, 1.0, 2.0, 5.0, 10.0)
TRANSLATIONS = (1.0, 2.0, 4.0)
AXES = 8


def scene(name):
    import torch
    from intrinsic3d_b200.scene import config_scene
    return config_scene(name, device="cuda:0" if torch.cuda.is_available() else "cpu")


def sdf0_engine(s):
    from intrinsic3d_b200 import engine
    e = engine.Engine(0)
    e.load_scene(s)
    return e, e.extract_mesh("fused", False)


def speed(name, gpu):
    from intrinsic3d_b200.scene import config_geometry, truth_mesh
    s = scene(name)
    e, m = sdf0_engine(s)
    truth = truth_mesh(**config_geometry(name))
    e.upload_reference_mesh(truth)
    e.register_reference_mesh()
    t0 = time.perf_counter()
    T, inf = e.register_reference_mesh()
    wall = time.perf_counter() - t0
    T2, inf2 = e.register_reference_mesh()
    n_sys = 31                               # the default schedule: 30 updates, then the system at the final pose
    tests = int(inf.point_triangle_tests)
    print(json.dumps({"metric": "register_device_ms", "workload": name, "gpu": gpu, "L": 1, "value": inf.ms_grid + inf.ms_rows + inf.ms_solve,
                      "unit": "ms", "wall_ms": 1e3 * wall, "resident_faces": len(m["faces"]), "truth_faces": len(truth["faces"]),
                      "status": inf.status, "iterations": inf.iterations, "systems": n_sys, "ms_grid": inf.ms_grid,
                      "ms_rows_per_system": inf.ms_rows / n_sys, "ms_solve_per_system": inf.ms_solve / n_sys,
                      "samples": int(inf.num_samples), "tests_per_sample": tests / (n_sys * inf.num_samples),
                      "tests_per_s": tests / (inf.ms_rows * 1e-3) if inf.ms_rows > 0 else None, "cell_size_m": inf.cell_size,
                      "grid": list(inf.grid), "cell_entries": int(inf.num_cell_entries),
                      "two_calls_same_bytes": T.tobytes() == T2.tobytes() and bytes(inf)[:-24] == bytes(inf2)[:-24],
                      "final_rms_vox": inf.final_rms / float(s["voxel_size"])}), flush=True)
    e.close()


def basin(name, gpu):
    import register_ref as rg
    s = scene(name)
    vs = float(s["voxel_size"])
    e, m = sdf0_engine(s)
    centre = np.asarray(m["vertices"], np.float64).mean(0)
    for deg in ROTATIONS:
        for tv in TRANSLATIONS:
            ok, rot, disp, status = 0, [], [], []
            for axis in range(AXES):
                G = rg.motion(deg, tv * vs, 1000 * axis + 7, centre)
                B = rg.moved(m, G)
                e.upload_reference_mesh(B)
                T, inf = e.register_reference_mesh()
                er, ed = rg.errors(T, rg.tr.inverse(list(G)), B["vertices"])
                rot.append(er); disp.append(ed / vs); status.append(int(inf.status))
                ok += int(er <= 1e-3 and ed <= 1e-3 * vs)
            print(json.dumps({"metric": "register_basin", "workload": name, "gpu": gpu, "rotation_deg": deg, "translation_vox": tv,
                              "converged_share": ok / AXES, "rot_err_deg": [float(x) for x in rot], "disp_err_vox": [float(x) for x in disp],
                              "status": status}), flush=True)
    e.close()


def odometry_engine(s, frames=25):
    import track_ref as tr
    from fusion_ref import depth_range, scene_inputs
    from intrinsic3d_b200 import engine
    dcam, depth, ccam, bgr, _, _ = scene_inputs(s)
    n = min(frames, int(depth.shape[0]))
    e = engine.Engine(0)
    e.sensor_frames_begin(dcam, ccam, int(depth.shape[0]))
    e.sensor_frames_add(depth, bgr)
    p = engine.default_fusion_params()
    p.voxel_size = float(s["voxel_size"])
    p.depth_min, p.depth_max = depth_range(s)
    e.fusion_begin(p)
    e.fusion_track_and_integrate_sensor(np.arange(n, dtype=np.int32), tr.aa_to_rt(s["poses_true"])[0])
    e.fusion_finish()
    return e


def quality(name, gpu):
    from intrinsic3d_b200.scene import config_geometry, truth_mesh
    s = scene(name)
    vs = float(s["voxel_size"])
    taus = [0.1 * vs, 0.25 * vs, 0.5 * vs]
    truth = truth_mesh(**config_geometry(name))

    def measure(e, label):
        e.upload_reference_mesh(truth)
        before = e.surface_distance(taus, 2 * vs, 2)
        T, inf = e.register_reference_mesh()
        e.transform_reference_mesh(T)
        after = e.surface_distance(taus, 2 * vs, 2)
        R = T[:9].reshape(3, 3)
        ang = math.degrees(math.acos(min(1.0, max(-1.0, (np.trace(R) - 1.0) * 0.5))))
        out = {"metric": "register_quality", "workload": name, "gpu": gpu, "row": label, "status": int(inf.status), "iterations": int(inf.iterations),
               "rotation_deg": ang, "translation_vox": float(np.linalg.norm(T[9:])) / vs, "T": [float(x) for x in T], "tau_vox": [0.1, 0.25, 0.5]}
        for k, r in (("before", before), ("after", after)):
            out[k] = {"accuracy_mean_vox": r["accuracy"]["mean"] / vs, "accuracy_rms_vox": r["accuracy"]["rms"] / vs,
                      "completeness_mean_vox": r["completeness"]["mean"] / vs, "completeness_rms_vox": r["completeness"]["rms"] / vs,
                      "fscore": r["fscore"]}
        print(json.dumps(out), flush=True)

    e, _ = sdf0_engine(s)
    measure(e, "1 sdf0")
    e.close()
    e = refined_engine(s)
    e.extract_mesh("refined", False)
    measure(e, "2 refined, 1 lighting estimate + 10 GN iterations")
    e.close()
    e = odometry_engine(s)
    e.extract_mesh("fused", False)
    measure(e, "3 fused from the first 25 frames by dense odometry")
    e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3")
    ap.add_argument("--basin", default="tiny,c2,c3")
    ap.add_argument("--skip-quality", action="store_true")
    args = ap.parse_args()
    gpu = gpu_info()
    for name in [w for w in args.workloads.split(",") if w]:
        speed(name, gpu)
    for name in [w for w in args.basin.split(",") if w]:
        basin(name, gpu)
    if not args.skip_quality:
        for name in [w for w in args.workloads.split(",") if w]:
            quality(name, gpu)


if __name__ == "__main__":
    main()
