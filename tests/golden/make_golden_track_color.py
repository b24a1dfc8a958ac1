"""Writes tests/golden/tiny_track_color.npz: the joint depth and colour tracking restatement tests/track_color_ref.py on the tiny scene fused
from its colour frames at the true poses, two frames from a seeded 1 cm / 1 deg perturbation.  Run from the repository root after
__graft_entry__.build()."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import track_color_ref as tc  # noqa: E402
import track_ref as tr  # noqa: E402
from test_track_color import tiny_fused  # noqa: E402

IDS, LEVELS, ITERATIONS = [2, 5], 2, (3, 2)


def main():
    s, dcam, depth, grid, rgb, inten, bgr = tiny_fused()
    pose_in = tr.perturb(tr.aa_to_rt(s["poses_true"]), 1.0, 0.01, seed=5)[IDS]
    fr = tc.track(grid, rgb, depth, inten, IDS, pose_in, dcam, num_levels=LEVELS, iterations=ITERATIONS)
    out = dict(ids=np.array(IDS, np.int32), num_levels=LEVELS, iterations=np.array(ITERATIONS, np.int32), dcam=np.array(dcam, np.float64),
               xyz=grid.xyz.astype(np.int32), sdf=grid.sdf, weight=grid.weight, voxel_size=np.float32(grid.vs), rgb=rgb, depth=depth, bgr=bgr,
               intensity=inten, pose_in=pose_in, model_intensity=np.stack([f.pint for f in fr]), sums=np.stack([f.sys for f in fr]),
               color_sums=np.stack([f.sys_c for f in fr]), outcome=np.array([[f.status, f.iterations, f.correspondences] for f in fr]),
               color_rows=np.array([[f.first[0], f.last[0]] for f in fr]), pose_out=np.array([f.w2c for f in fr]))
    for l in range(LEVELS):
        out[f"intensity_{l}"] = np.stack([f.inten[l] for f in fr])
        out[f"grad_x_{l}"] = np.stack([f.grads[l][0] for f in fr])
        out[f"grad_y_{l}"] = np.stack([f.grads[l][1] for f in fr])
    np.savez_compressed(os.path.join(HERE, "tiny_track_color.npz"), **out)


if __name__ == "__main__":
    main()
