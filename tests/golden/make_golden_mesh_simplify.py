"""Writes tests/golden/tiny_mesh_simplify.npz: the refined, largest-component mesh of the tiny_mesh.npz fixture and its simplifications
by tests/mesh_simplify_ref.py at cells of 2 and 4 voxels, and the 2-voxel result simplified again at 4 voxels (chained).

    python tests/golden/make_golden_mesh_simplify.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import mesh_ref  # noqa: E402
import mesh_simplify_ref as msr  # noqa: E402


def main():
    g = np.load(os.path.join(HERE, "tiny_mesh.npz"))
    vs = float(g["voxel_size"])
    m = mesh_ref.extract(g["xyz"], g["sdf_refined"], g["weight"], g["rgb"], vs, True)
    for k in ("vertices", "colors", "faces"):
        assert m[k].tobytes() == g[f"refined_1_{k}"].tobytes()
    cells = np.array([2 * vs, 4 * vs, 4 * vs], np.float32)
    chained = np.array([False, False, True])
    out = dict(in_vertices=m["vertices"], in_colors=m["colors"], in_faces=m["faces"], voxel_size=np.float32(vs), cells=cells, chained=chained)
    prev = None
    for k, cell in enumerate(cells):
        s = msr.simplify(prev if chained[k] else m, float(cell))
        for key in ("vertices", "colors", "faces"):
            out[f"{k}_{key}"] = s[key]
        out[f"{k}_info"] = np.array([s["info"][c] for c in msr.INFO_COUNTS], np.int64)
        print(k, float(cell), s["info"])
        prev = s
    np.savez_compressed(os.path.join(HERE, "tiny_mesh_simplify.npz"), **out)


if __name__ == "__main__":
    main()
