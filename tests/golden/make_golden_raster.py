"""Writes tests/golden/tiny_raster.npz: the tiny scene's refined, largest-component mesh (voxel colours) rasterized by tests/raster_ref.py
into keyframes 0, 2 and 5 with the engine camera and vertex colours, with the statistics against the scene's depth and
make_color_frames.

    python tests/golden/make_golden_raster.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import mesh_ref  # noqa: E402
import raster_ref as ra  # noqa: E402
import render_ref as rr  # noqa: E402
from intrinsic3d_b200.scene import config_scene, make_color_frames  # noqa: E402


def main():
    s = config_scene("tiny")
    col = make_color_frames(s)
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], s["rgb"], float(s["voxel_size"]), True)
    ids = np.array([0, 2, 5], np.int32)
    _, H, W = s["depth"].shape
    r = ra.rasterize(m, rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"]), W, H, color="vertex", depth=s["depth"], bgr=col, ids=ids)
    out = dict(faces=m["faces"].astype(np.int32), ids=ids, **{k: r[k] for k in ra.PLANES})
    out["counts"] = np.array([[st["num_covered"], st["num_observed"], st["depth_count"], st["color_count"], *st["color_abs"], *st["color_sq"]]
                              for st in r["stats"]], np.int64)
    out["sums"] = np.array([[st["depth_abs"], st["depth_sq"]] for st in r["stats"]], np.float64)
    np.savez_compressed(os.path.join(HERE, "tiny_raster.npz"), **out)
    print(r["stats"])


if __name__ == "__main__":
    main()
