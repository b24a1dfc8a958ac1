"""Writes tests/golden/tiny_distance.npz: the distance of the tiny scene's refined, largest-component mesh to its truth_mesh (n_theta
32) computed by tests/distance_ref.py at L = 2, max_distance 2 voxels, thresholds 0.1, 0.25 and 0.5 voxel: per-sample and per-vertex
(d^2, face) and the statistics.

    python tests/golden/make_golden_distance.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import distance_ref as dr  # noqa: E402
import mesh_ref  # noqa: E402
from intrinsic3d_b200.scene import config_geometry, config_scene, truth_mesh  # noqa: E402

L, N_THETA = 2, 32


def inputs():
    s = config_scene("tiny")
    vs = float(s["voxel_size"])
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], s["rgb"], vs, True)
    return m, truth_mesh(N_THETA, **config_geometry("tiny")), 2 * vs, [0.1 * vs, 0.25 * vs, 0.5 * vs]


def main():
    m, t, maxd, taus = inputs()
    r = dr.distance(m, t, L, maxd, taus)
    out = dict(faces=m["faces"], truth_faces=t["faces"], L=np.int32(L), max_distance=np.float32(maxd), thresholds=np.array(taus, np.float32))
    for k in ("accuracy_d2", "accuracy_face", "completeness_d2", "completeness_face", "vertex_distance", "vertex_face"):
        out[k] = r[k]
    for k in ("accuracy", "completeness"):
        out[k + "_stats"] = np.array([r[k][c] for c in ("mean", "rms", "max", "area", "unmatched_area")] + r[k]["fraction"], np.float64)
    out["fscore"] = np.array(r["fscore"], np.float64)
    np.savez_compressed(os.path.join(HERE, "tiny_distance.npz"), **out)
    print(len(m["faces"]), len(t["faces"]), r["accuracy"]["mean"], r["completeness"]["mean"], r["fscore"])


if __name__ == "__main__":
    main()
