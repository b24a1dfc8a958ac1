"""Generates tests/golden/tiny_render.npz: a small constructed scene (a sphere with noisy sdf, a few zero-weight voxels, per-voxel SH,
two views with lens distortion, frames with holes) and what tests/render_ref.py renders of it: planes and statistics per view.

    python tests/golden/make_golden_render.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import render_ref as rr  # noqa: E402

STATS = ("num_hit", "num_observed", "depth_count", "photo_count", "depth_abs", "depth_sq", "photo_abs", "photo_sq")


def scene():
    rng = np.random.default_rng(11)
    vs = np.float32(0.01)
    r = np.arange(-9, 10)
    X, Y, Z = np.meshgrid(r, r, r, indexing="ij")
    xyz = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1).astype(np.int32)
    d = np.linalg.norm(xyz.astype(np.float64), axis=1) * float(vs) - 0.06
    keep = np.abs(d) <= 3 * float(vs)
    xyz, d = xyz[keep], d[keep]
    n = len(xyz)
    sdf = d + rng.normal(0.0, 0.1 * float(vs), n)
    albedo = 0.5 + 0.3 * rng.random(n)
    weight = np.where(rng.random(n) < 0.02, 0.0, 1.0).astype(np.float32)
    sh = np.tile([0.8, 0.1, -0.2, 0.15, 0.02, -0.03, 0.05, 0.01, -0.04], (n, 1)) + 0.02 * rng.standard_normal((n, 9))
    sh_has = np.ones(n, np.uint8)          # as i3d_set_sh installs them (partial SH comes from the lighting estimate)
    W, H = 40, 32
    poses = np.array([[0.0, 0.0, 0.0, 0.0, 0.0, 0.25], [0.1, -0.4, 0.05, 0.02, -0.01, 0.27]])
    intr = np.array([45.0, 46.0, 19.3, 15.6])
    dist = np.array([0.05, -0.02, 0.0, 0.001, -0.002])
    depth = (0.2 + 0.05 * rng.random((2, H, W))).astype(np.float32)
    depth[rng.random((2, H, W)) < 0.1] = 0.0
    lum = rng.random((2, H, W)).astype(np.float32)
    return dict(xyz=xyz, sdf0=-sdf, sdf_refined=sdf, albedo=albedo, weight=weight, rgb=np.full((n, 3), 100, np.uint8), voxel_size=vs, sh=sh,
                sh_has=sh_has, poses=poses, intr=intr, dist=dist, depth=depth, lum=lum)


def compute():
    s = scene()
    grid = rr.grid_of(s, "refined", s["sh"], s["sh_has"])
    out = rr.render(grid, s["poses"], s["intr"], s["dist"], 1.0, [0, 1], s["depth"], s["lum"])
    res = {k: v for k, v in s.items()}
    for p in rr.PLANES:
        res["plane_" + p] = out[p]
    res["stats_int"] = np.array([[st[k] for k in STATS[:4]] for st in out["stats"]], np.int64)
    res["stats_sum"] = np.array([[st[k] for k in STATS[4:]] for st in out["stats"]], np.float64)
    return res


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "tiny_render.npz"), **compute())
    print("wrote tiny_render.npz")
