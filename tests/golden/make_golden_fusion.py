"""Generates tests/golden/tiny_fusion.npz: the inputs of a 3-frame RGB-D fusion of a small seeded scene (depth, colour, float poses in
both directions, camera, fusion parameters) and the fusion oracle's result after correctSDF (Jacobi) and clearInvalidVoxels.  The
inputs are stored so that the fixture does not depend on the scene generator.  Needs tests/native/libfusion_oracle.so
(__graft_entry__.build()).   Run:  python tests/golden/make_golden_fusion.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))


def main():
    from fusion_ref import FusionOracle, depth_range, scene_inputs
    from intrinsic3d_b200.scene import make_scene
    s = make_scene(radius_vox=10.0, frames=3, width=96, height=72, voxel_size=0.004, seed=2)
    cam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    dmin, dmax = depth_range(s)
    params = np.array([float(s["voxel_size"]), dmin, dmax, 10.0], np.float32)
    o = FusionOracle(voxel_size=params[0], depth_min=params[1], depth_max=params[2], weight_sample=params[3], window=2, iterations=10)
    assert o.integrate(cam, depth, ccam, bgr, c2w, w2c) == 0
    sweeps = o.finish(1)
    v = o.volume()
    np.savez_compressed(os.path.join(HERE, "tiny_fusion.npz"), cam=np.array(cam, np.float64), depth=depth, bgr=bgr, c2w=c2w, w2c=w2c,
                        params=params, sweeps=np.int32(sweeps), **v)
    print(f"tiny_fusion.npz: {len(v['xyz'])} voxels, {sweeps} sweeps")


if __name__ == "__main__":
    main()
