"""Writes tests/golden/tiny_odometry.npz: the odometry restatement of tests/test_odometry.py on the first frames of the dense tiny
sequence (5 degrees of orbit per frame), frame 0 anchored at its true pose.  Run from the repository root after __graft_entry__.build()."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import track_ref as tr  # noqa: E402
from test_odometry import dense_tiny, run_sequence  # noqa: E402

FRAMES, IDS, ITERATIONS = 72, [0, 1, 2, 3, 4, 5], (4, 2, 2)


def main():
    s = dense_tiny(FRAMES)
    pose_first = tr.aa_to_rt(s["poses_true"])[0]
    odo = run_sequence(s, IDS, pose_first, iterations=ITERATIONS)
    v = odo.volume()
    np.savez_compressed(os.path.join(HERE, "tiny_odometry.npz"), frames=FRAMES, ids=np.array(IDS, np.int32), pose_first=pose_first,
                        iterations=np.array(ITERATIONS, np.int32), status=np.array([f[0] for f in odo.frames], np.int32),
                        pose_out=np.array([f[1] for f in odo.frames]), **{f"volume_{k}": v[k] for k in v})


if __name__ == "__main__":
    main()
