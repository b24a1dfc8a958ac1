"""Generates tests/golden/tiny_sensor.npz: two depth frames of the fusion tests' scene (stored, so that the fixture does not depend on the
scene generator), their depth camera, the fusion tests' colour camera at twice the size, and the planes tests/sensor_ref.py resizes them to.
Run:  python tests/golden/make_golden_sensor.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))


def main():
    import sensor_ref
    from intrinsic3d_b200.scene import make_scene
    s = make_scene(radius_vox=16.0, frames=5, width=160, height=120, voxel_size=0.004, seed=3)
    F, H, W = s["depth"].shape
    dcam = (W, H, *(float(v) for v in s["intr"]))
    ccam = sensor_ref.color_cameras(dcam)["color_x2"]
    depth = np.ascontiguousarray(s["depth"][:2], np.float32)
    out = sensor_ref.resize_depth(depth, dcam, ccam)
    print(depth.shape, "->", out.shape, int((out > 0).sum()), "pixels with depth")
    np.savez_compressed(os.path.join(HERE, "tiny_sensor.npz"), depth=depth, depth_cam=np.array(dcam, np.float64),
                        color_cam=np.array(ccam, np.float64), resized=out)


if __name__ == "__main__":
    main()
