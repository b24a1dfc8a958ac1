"""Generates tests/golden/tiny_mesh.npz: the tiny scene's grid (stored, so that the fixture does not depend on the scene generator) and
the meshes tests/mesh_ref.py extracts from it, for both sdf sources with and without the component filter.
Run:  python tests/golden/make_golden_mesh.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))


def main():
    import mesh_ref
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("tiny")
    g = dict(xyz=s["xyz"].astype(np.int32), sdf0=s["sdf0"].astype(np.float64), sdf_refined=s["sdf_refined"].astype(np.float64),
             weight=s["weight"].astype(np.float32), rgb=s["rgb"].astype(np.uint8), voxel_size=np.float32(s["voxel_size"]))
    out = dict(g)
    for src in ("fused", "refined"):
        for lc in (0, 1):
            m = mesh_ref.extract_grid(g, src, bool(lc))
            for k in ("vertices", "colors", "faces"):
                out[f"{src}_{lc}_{k}"] = m[k]
            print(src, lc, m["info"])
    np.savez_compressed(os.path.join(HERE, "tiny_mesh.npz"), **out)


if __name__ == "__main__":
    main()
