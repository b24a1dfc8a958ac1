"""Writes tests/golden/tiny_grid_from_mesh.npz: the tiny scene's truth mesh at 32 rings and the grid the numpy restatement
(tests/grid_from_mesh_ref.py) converts it to at the scene's voxel size, band 3: xyz, sdf, nearest face and feature per voxel."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import grid_from_mesh_ref as gr  # noqa: E402
from intrinsic3d_b200.scene import config_geometry, truth_mesh  # noqa: E402


def main():
    geo = config_geometry("tiny")
    mesh = truth_mesh(32, **geo)
    vs, band = np.float32(geo["voxel_size"]), np.float32(3.0)
    out = gr.grid_from_mesh(mesh, float(vs), float(band))
    np.savez_compressed(os.path.join(HERE, "tiny_grid_from_mesh.npz"), vertices=mesh["vertices"], faces=mesh["faces"], voxel_size=vs, band=band,
                        xyz=out["xyz"], sdf=out["sdf"], face=out["face"], feature=out["feature"])
    print(len(out["xyz"]), "voxels", (out["sdf"] < 0).sum(), "negative")


if __name__ == "__main__":
    main()
