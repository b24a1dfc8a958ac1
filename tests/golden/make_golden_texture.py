"""Writes tests/golden/tiny_texture.npz: the texture of the tiny scene's refined, largest-component mesh (voxel colours of the scene,
engine camera, make_color_frames) baked by tests/texture_ref.py at (S, K) = (8, 5), (6, 0) and (7, 1).

    python tests/golden/make_golden_texture.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import mesh_ref  # noqa: E402
import render_ref as rr  # noqa: E402
import texture_ref as tr  # noqa: E402
from intrinsic3d_b200.scene import config_scene, make_color_frames  # noqa: E402


def main():
    s = config_scene("tiny")
    col = make_color_frames(s)
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], s["rgb"], float(s["voxel_size"]), True)
    cases = np.array([[8, 5], [6, 0], [7, 1]], np.int32)
    out = dict(faces=m["faces"], occlusion=np.float32(0.02), cases=cases)
    for k, (S, K) in enumerate(cases):
        b = tr.bake(m, s["depth"], col, rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"]), int(S), 0.02, int(K))
        out[f"{k}_image"], out[f"{k}_uv"] = b["image"], b["uv"]
        out[f"{k}_info"] = np.array([b["info"][c] for c in tr.INFO_COUNTS], np.int64)
        print(k, S, K, b["info"])
    np.savez_compressed(os.path.join(HERE, "tiny_texture.npz"), **out)


if __name__ == "__main__":
    main()
