"""Writes tests/golden/tiny_intrinsic_texture.npz: the tiny scene's refined, largest-component mesh (voxel colours), its S = 6 texture
from all keyframes (tests/texture_ref.py, engine camera, K = 5), and its decomposition by tests/intrinsic_texture_ref.py under a global
SH and under the oracle's lighting estimate (sub_index, sub_sh, subvolume_size stored; that case's albedo and shading by their
SHA-256), with the relit keyframes 1 and 4 under the
global SH.

    python tests/golden/make_golden_intrinsic_texture.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import intrinsic_texture_ref as it  # noqa: E402
import mesh_ref  # noqa: E402
import oracle  # noqa: E402
import render_ref as rr  # noqa: E402
import texture_ref as tr  # noqa: E402
from intrinsic3d_b200.scene import config_scene, make_color_frames  # noqa: E402

S = 6
SH = np.array([0.75, 0.1, -0.2, 0.15, 0.04, -0.05, 0.06, 0.02, -0.03], np.float32)
MIN_SHADING = 0.05


def main():
    s = config_scene("tiny")
    col = make_color_frames(s)
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], s["rgb"], float(s["voxel_size"]), True)
    rt, cam = rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"])
    b = tr.bake(m, s["depth"], col, rt, cam, S, 0.02, 5)
    obs = it.observed(m, s["depth"], rt, cam, S)
    o = oracle.Oracle(threads=4)
    o.set_grid(s)
    lp = oracle.default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    o.estimate_lighting(lp)
    idx, sub = o.lighting()
    out = dict(faces=m["faces"].astype(np.int32), image=b["image"], observed=obs, sh=SH, min_shading=np.float32(MIN_SHADING),
               sub_index=idx, sub_sh=sub, subvolume_size=np.float32(lp.subvolume_size))
    for name, light in (("global", it.global_sh(SH)), ("estimate", it.estimate_sh(idx, sub, float(lp.subvolume_size)))):
        d = it.decompose(b["image"], m, S, light, MIN_SHADING, obs)
        if name == "global":
            out["global_albedo"], out["global_shading"] = d["albedo"], d["shading"]
        else:                       # the second case by digest, to keep the file small
            out["estimate_digest"] = np.frombuffer(hashlib.sha256(d["albedo"].tobytes() + d["shading"].tobytes()).digest(), np.uint8)
        out[f"{name}_info"] = np.array([d["info"][k] for k in it.INFO_COUNTS], np.int64)
        out[f"{name}_range"] = np.array([d["info"]["albedo_min"], d["info"]["albedo_max"]], np.float32)
        print(name, d["info"])
    ids = np.array([1, 4], np.int32)
    _, H, W = s["depth"].shape
    r = it.rasterize(m, rt, cam, W, H, out["global_albedo"], S, it.global_sh(SH), depth=s["depth"], bgr=col, ids=ids)
    out["relit_ids"], out["relit_rgb"], out["relit_face"] = ids, r["rgb"], r["face"]
    out["relit_counts"] = np.array([[st["num_covered"], st["color_count"], *st["color_abs"], *st["color_sq"]] for st in r["stats"]], np.int64)
    np.savez_compressed(os.path.join(HERE, "tiny_intrinsic_texture.npz"), **out)


if __name__ == "__main__":
    main()
