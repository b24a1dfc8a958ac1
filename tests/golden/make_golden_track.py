"""Writes tests/golden/tiny_track.npz: two frames of the tiny scene tracked by the restatement tests/track_ref.py against sdf0 from the
scene's perturbed poses (2 pyramid levels, iterations {2, 1}).  Holds the grid, the depth frames and the input poses, and per frame the
pyramid and normal planes, the prediction planes, the last level-0 correspondence mask, the last system's sums, the outcome and the pose.

    python tests/golden/make_golden_track.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import render_ref as rr  # noqa: E402
import track_ref as tr  # noqa: E402
from intrinsic3d_b200.scene import config_scene  # noqa: E402


def main():
    s = config_scene("tiny")
    ids = np.array([1, 4], np.int32)
    F, H, W = s["depth"].shape
    dcam = np.array([W, H] + [float(v) for v in s["intr"]], np.float64)
    pose_in = tr.aa_to_rt(s["poses"])[ids]
    levels, iters = 2, np.array([2, 1, 0, 0], np.int32)
    grid = rr.Grid(s["xyz"], s["sdf0"], s["albedo"], s["weight"], s["voxel_size"])
    depth = np.ascontiguousarray(s["depth"][:5], np.float32)
    fr = tr.track(grid, depth, ids.tolist(), pose_in, tuple(dcam), num_levels=levels, iterations=iters.tolist())
    out = dict(xyz=s["xyz"], sdf0=s["sdf0"], sdf_refined=s["sdf_refined"], albedo=s["albedo"], weight=s["weight"], rgb=s["rgb"],
               voxel_size=s["voxel_size"], depth=depth, ids=ids, dcam=dcam, pose_in=pose_in, num_levels=np.int32(levels), iterations=iters,
               pred_depth=np.stack([f.pdepth for f in fr]), pred_normal=np.stack([f.pnrm for f in fr]), mask=np.stack([f.mask for f in fr]),
               sums=np.stack([f.sys for f in fr]), outcome=np.array([[f.status, f.iterations, f.correspondences] for f in fr], np.int64),
               pose_out=np.array([f.w2c for f in fr]),
               initial=np.array([[f.initial[k] for k in ("num_hit", "num_observed", "depth_count", "depth_abs", "depth_sq")] for f in fr]))
    for l in range(levels):
        out[f"depth_{l}"] = np.stack([f.depth[l] for f in fr])
        out[f"normal_{l}"] = np.stack([f.nrm[l] for f in fr])
    np.savez_compressed(os.path.join(HERE, "tiny_track.npz"), **out)
    print("wrote tiny_track.npz:", [(f.status, f.iterations, f.correspondences) for f in fr])


if __name__ == "__main__":
    main()
