#!/usr/bin/env python
"""bench_intrinsic_texture.py — the texture decomposition (i3d_decompose_texture) and the relit raster source on the C3 grid, one JSON line.

    python bench_intrinsic_texture.py [--workload c3|c2|small|tiny] [--reps 5] [--gn 4] [--quality c2,c3]

Speed: after a lighting estimate (default parameters, S subvolumes as the estimate makes them), the workload's refined mesh without the
component filter, full and simplified at cells of 2, 4 and 8 voxels, baked at 12 texels per face (K = 5).  Per mesh, the median of --reps
calls after one warm-up call of: the bake (ms_bake) and its observation flags (phase "texture_observed"); the decomposition under the
estimate and under a global SH (ms_decompose); the statistics of every keyframe with the texture source and with the relit source
(planes=(), device ms per stage).

Byte model of k_tex_decompose, kept here: per atlas texel 3 B of baked colour, 1 B of observation flag, 12 B of albedo and 4 B of shading
written; per owned texel 12 B of face indices and 36 B of vertex positions.  The estimate's subvolume table and SH (a few KB, read by
every texel) stay in cache and are left out.  Reported as GB/s of that model against the H100 SXM data sheet's 3350 GB/s.

Quality (--quality): per scene, --gn Gauss-Newton iterations refine the albedo, then the lighting is estimated, the refined mesh (4-voxel
simplification) is baked at 12 texels per face and decomposed under the estimate (and, for a scene with one global SH, under the true SH).
Per owned lit texel the true albedo at the radially closest surface point is compared with the channel mean of A_k / g_k (g = the
channel gains of make_color_frames) after one least-squares scale; the same for the colour texture itself (c / 255 / g) and for the
refined per-vertex `albedo` colour mode blended at the texel.  Reported: mean absolute error and scale per estimate.  The GPU name and
power limit are read in the same run.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
PEAK_GBS = 3350.0
G = np.array([1.00, 0.92, 0.85])
SH_GLOBAL = np.array([0.8, 0.1, -0.1, 0.15, 0.02, -0.03, 0.04, 0.01, -0.02], np.float32)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return out.stdout.strip() or None
    except Exception:
        return None


def decompose_bytes(texels, owned):
    return 20 * texels + 48 * owned


def lighting(e, s, engine):
    lp = engine.default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    e.estimate_lighting(lp)
    return float(lp.subvolume_size)


def speed(e, vs, cell, reps):
    m = e.extract_mesh("refined", False)
    if cell:
        m = e.simplify_mesh(cell * vs)
    bake, obs = [], []
    for _ in range(reps + 1):
        b = e.bake_texture(12)
        bake.append(b["info"].ms_bake)
        obs.append(e.phase_ms("texture_observed"))
    i = b["info"]
    texels = int(i.atlas_width) * int(i.atlas_height)
    out = {"cell_voxels": cell or 0, "faces": int(i.num_faces), "texels": texels, "owned": int(i.num_texels_owned),
           "fallback": int(i.num_texels_fallback), "ms_bake": float(np.median(bake[1:])), "ms_observed_flags": float(np.median(obs[1:]))}
    for name, sh in (("estimate", None), ("global", SH_GLOBAL)):
        ms = [e.decompose_texture(0.05, sh)["info"].ms_decompose for _ in range(reps + 1)][1:]
        d = float(np.median(ms))
        gbs = decompose_bytes(texels, out["owned"]) / (d * 1e-3) / 1e9
        out[f"decompose_{name}"] = {"device_ms": d, "model_gbs": gbs, "share_of_3350": gbs / PEAK_GBS}
    ids = list(range(e.F))
    e.set_relight(None)
    for src in ("texture", "relit"):
        e.rasterize_keyframes(ids, src, planes=())
        runs = []
        for _ in range(reps):
            t0 = time.perf_counter()
            r = e.rasterize_keyframes(ids, src, planes=())
            runs.append((1e3 * (time.perf_counter() - t0), r["info"]))
        med = lambda k: float(np.median([getattr(x[1], k) for x in runs]))
        st = r["stats"]
        n = max(1, sum(x["color_count"] for x in st))
        out[f"raster_{src}"] = {"views": len(ids), "ms_rays": med("ms_rays"), "ms_faces": med("ms_faces"), "ms_shade": med("ms_shade"),
                                "device_ms": med("ms_rays") + med("ms_faces") + med("ms_shade"), "wall_ms": float(np.median([x[0] for x in runs])),
                                "color_mae": [sum(x["color_abs"][k] for x in st) / n for k in range(3)]}
    return out


def _fit(est, truth):
    alpha = float((est * truth).sum() / (truth * truth).sum())
    return {"mae": float(np.abs(est / alpha - truth).mean()), "scale": alpha}


def quality(name, device, gn):
    import texture_ref as tr
    import torch
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200 import scene as sc
    s = sc.config_scene(name, device=device)
    e = engine.Engine(0)
    e.load_scene(s)
    e.upload_color_frames(sc.make_color_frames(s))
    p = engine.default_params()
    p.thres_shell = s["thres_shell"]
    for _ in range(gn):
        e.gn_iteration(p)
    lighting(e, s, engine)
    vs = float(np.float32(s["voxel_size"]))
    e.extract_mesh("refined", False, "albedo")
    m_alb = e.simplify_mesh(4 * vs)                      # the per-vertex albedo mode on the same mesh
    e.extract_mesh("refined", False)
    m = e.simplify_mesh(4 * vs)
    assert m["faces"].tobytes() == m_alb["faces"].tobytes()
    b = e.bake_texture(12)
    tp = tr.texel_points(m, 12)
    geo = sc.config_geometry(name)
    rho0, bump = float(geo["radius_vox"]) * vs, 0.03
    P = torch.tensor(tp["P"].astype(np.float64))
    d = P / torch.linalg.norm(P, dim=-1, keepdim=True)
    ps = d * sc._rho(d, rho0, bump)[..., None]
    truth = sc._albedo_truth(ps, max(6.0 * vs, rho0 / 4.0)).numpy()
    ests = {"decomposition_estimate": e.decompose_texture(0.05)["albedo"]}
    sh = np.asarray(s["sh"].cpu() if hasattr(s["sh"], "cpu") else s["sh"], np.float64).reshape(-1, 9)
    if np.all(sh == sh[0]):
        ests["decomposition_true_sh"] = e.decompose_texture(0.05, sh[0].astype(np.float32))["albedo"]
    lit = np.ones(len(truth), bool)
    for a in ests.values():
        lit &= a[tp["y"], tp["x"]].any(1)
    out = {k: _fit((a[tp["y"], tp["x"]].astype(np.float64) / G).mean(1)[lit], truth[lit]) for k, a in ests.items()}
    out["colour_texture"] = _fit((b["image"][tp["y"], tp["x"]].astype(np.float64) / 255.0 / G).mean(1)[lit], truth[lit])
    fv = m["faces"][tp["face"]]
    vc = m_alb["colors"].astype(np.float64).mean(1) / 255.0
    vert = sum(w.astype(np.float64) * vc[fv[:, q]] for q, w in enumerate((tp["w0"], tp["a"], tp["b"])))
    out["vertex_albedo_mode"] = _fit(vert[lit], truth[lit])
    out.update(scene=name, faces=len(m["faces"]), lit_texels=int(lit.sum()), gn_iterations=gn, sh_varying=bool(not np.all(sh == sh[0])))
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=["tiny", "small", "c2", "c3"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--gn", type=int, default=4)
    ap.add_argument("--quality", default="c2,c3")
    args = ap.parse_args()

    import torch
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    sys.path.insert(0, os.path.join(ROOT, "tests"))

    gpu = gpu_info()
    device = "cuda:0" if torch.cuda.is_available() else "cpu"
    scene = config_scene(args.workload, device=device)
    e = engine.Engine(0)
    e.load_scene(scene)
    e.upload_color_frames(make_color_frames(scene))
    lighting(e, scene, engine)
    reps = max(1, args.reps)
    vs = float(np.float32(scene["voxel_size"]))
    runs = [speed(e, vs, cell, reps) for cell in (None, 2, 4, 8)]
    e.close()
    q = [quality(n, device, args.gn) for n in args.quality.split(",") if n]
    line = {"metric": "decompose_texture_device_ms", "value": runs[0]["decompose_estimate"]["device_ms"], "unit": "ms", "higher_is_better": False,
            "workload": args.workload, "gpu": gpu, "reps": reps, "runs": runs, "quality": q, "peak_gbs": PEAK_GBS}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
