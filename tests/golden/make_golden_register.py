"""Writes tests/golden/tiny_register.npz: the tiny scene's sdf0 mesh as the resident mesh and a copy moved by 2 degrees and 1 voxel as the
reference, registered by tests/register_ref.py at L = 1 with stages (0.016, 0.008) m of 3 iterations each: every system, the pose each was
formed at, the per-sample nearest face at the initial pose, the returned T and the status.

    python tests/golden/make_golden_register.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import mesh_ref  # noqa: E402
import register_ref as rg  # noqa: E402
from intrinsic3d_b200.scene import config_scene  # noqa: E402

STAGES = dict(max_distance=(0.016, 0.008), iterations=(3, 3), samples_per_edge=1)


def inputs():
    s = config_scene("tiny")
    vs = float(s["voxel_size"])
    A = mesh_ref.extract(s["xyz"], s["sdf0"], s["weight"], s["rgb"], vs, True)
    G = rg.motion(2.0, vs, 11, np.asarray(A["vertices"], np.float64).mean(0))
    return A, rg.moved(A, G), G


def main():
    A, B, G = inputs()
    out = rg.register(A, B, **STAGES)
    f0 = rg.rows(A, B, rg.tr.inverse(rg.IDENTITY), 1, np.float32(STAGES["max_distance"][0]), np.float32(0.5))["face"]
    np.savez_compressed(os.path.join(HERE, "tiny_register.npz"), a_vertices=A["vertices"], a_faces=A["faces"], b_vertices=B["vertices"],
                        G=G, systems=out["systems"], poses=out["Ms"], faces0=f0, T=out["T"], status=np.int32(out["status"]),
                        iterations=np.int32(out["iterations"]))
    print(len(A["faces"]), out["status"], out["iterations"], out["T"])


if __name__ == "__main__":
    main()
