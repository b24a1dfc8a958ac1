"""Generates tests/golden/tiny_vis.npz: a grid made from the tiny scene (stored, so that the fixture does not depend on the scene
generator), the subvolume SH of the CPU oracle's lighting estimate on it, and the colours tests/vis_ref.py gives for every colour mode and
both sdf sources.  The refined sdf and the albedo are perturbed (seeded) so that the sources differ and the albedo varies.
Run (after __graft_entry__.build(), which builds the oracle):  python tests/golden/make_golden_vis.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

SUBVOLUME_SIZE = 0.02


def main():
    import oracle
    import vis_ref
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("tiny")
    rng = np.random.default_rng(11)
    vs = float(s["voxel_size"])
    sdf0 = s["sdf0"].astype(np.float64)
    s = dict(s)
    s["sdf_refined"] = sdf0 + rng.normal(0.0, 0.2 * vs, len(sdf0))
    s["albedo"] = np.clip(0.6 + 0.25 * rng.standard_normal(len(sdf0)), 0.0, 1.2)
    o = oracle.Oracle(threads=4)
    o.load_scene(s)
    lp = oracle.default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    lp.subvolume_size = SUBVOLUME_SIZE
    o.estimate_lighting(lp)
    sub_index, sub_sh = o.lighting()
    g = dict(xyz=s["xyz"].astype(np.int32), sdf0=sdf0, sdf_refined=s["sdf_refined"].astype(np.float64), albedo=s["albedo"].astype(np.float64),
             weight=s["weight"].astype(np.float32), rgb=s["rgb"].astype(np.uint8), voxel_size=np.float32(s["voxel_size"]))
    out = dict(g, sub_index=np.asarray(sub_index, np.int32), sub_sh=np.asarray(sub_sh, np.float64), subvolume_size=np.float32(SUBVOLUME_SIZE))
    for src in ("fused", "refined"):
        for mode in vis_ref.MODES:
            out[f"{src}_{mode or 'voxel'}"] = vis_ref.colors(g, mode, src, out["sub_index"], out["sub_sh"], SUBVOLUME_SIZE)
    print(len(g["xyz"]), "voxels,", len(sub_sh), "subvolumes")
    np.savez_compressed(os.path.join(HERE, "tiny_vis.npz"), **out)


if __name__ == "__main__":
    main()
