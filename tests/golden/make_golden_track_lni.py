"""Writes tests/golden/tiny_track_lni.npz: the LNI restatement tests/track_lni_ref.py on the tiny scene fused from its colour frames at the
true poses, two frames from a seeded 1 cm / 1 deg perturbation, frame 2 referenced to frame 1 and frame 5 to itself, at their true poses,
with norm_radius 5 and norm_eps 0.01.  Run from the repository root after __graft_entry__.build()."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import track_lni_ref as tl  # noqa: E402
import track_ref as tr  # noqa: E402
from test_track_color import tiny_fused  # noqa: E402

IDS, REFS, LEVELS, ITERATIONS = [2, 5], [1, 5], 3, (3, 2, 2)
RADIUS, EPS = 5, 0.01


def main():
    s, dcam, depth, grid, rgb, inten, bgr = tiny_fused()
    true = tr.aa_to_rt(s["poses_true"])
    pose_in = tr.perturb(true, 1.0, 0.01, seed=5)[IDS]
    ref_pose = true[REFS]
    fr = tl.track(grid, depth, inten, IDS, pose_in, REFS, ref_pose, dcam, color=dict(norm_radius=RADIUS, norm_eps=EPS), num_levels=LEVELS,
                  iterations=ITERATIONS)
    out = dict(ids=np.array(IDS, np.int32), ref_ids=np.array(REFS, np.int32), num_levels=LEVELS, iterations=np.array(ITERATIONS, np.int32),
               norm_radius=np.int32(RADIUS), norm_eps=np.float32(EPS),
               dcam=np.array(dcam, np.float64), xyz=grid.xyz.astype(np.int32), sdf=grid.sdf, weight=grid.weight, voxel_size=np.float32(grid.vs),
               rgb=rgb, depth=depth, bgr=bgr, intensity=inten, pose_in=pose_in, ref_pose=ref_pose, sums=np.stack([f.sys for f in fr]),
               color_sums=np.stack([f.sys_c for f in fr]), outcome=np.array([[f.status, f.iterations, f.correspondences] for f in fr]),
               color_rows=np.array([[f.first[0], f.last[0]] for f in fr]), pose_out=np.array([f.w2c for f in fr]))
    for l in range(LEVELS):
        out[f"model_{l}"] = np.stack([f.models[l] for f in fr])
        out[f"ref_intensity_{l}"] = np.stack([f.ref_inten[l] for f in fr])
        out[f"intensity_{l}"] = np.stack([f.inten[l] for f in fr])
    np.savez_compressed(os.path.join(HERE, "tiny_track_lni.npz"), **out)


if __name__ == "__main__":
    main()
