"""BASELINE.json config 5: the coarse-to-fine schedule of Intrinsic3D::refine (src/refinement/intrinsic3d.cpp:206-295) end to end on
N GPUs:  3 grid levels (4 mm -> 2 mm -> 1 mm: ~0.5 M -> ~2 M -> ~8 M voxels after thin-shell pruning), 500 frames 640x480, all 3 pyramid
levels on the coarsest grid only => 5 Optimizer::optimize calls x 10 GN iterations = 50 GN iterations per refinement, each call preceded
by the SVSH lighting estimate and followed by the voxel recolouring; pruning before every grid level, x2 upsampling after.

Called by `bench.py --workload c5`.  One step = ONE whole refinement through the C-ABI; `value` = GN iterations / second over the whole
schedule (everything the schedule does is inside the timed region: grid upload, frame uploads at pyramid-level switches, lighting,
recolouring, pruning, upsampling, shard setup).  Multi-GPU: the GN iterations are voxel-sharded; lighting / recolouring / grid
transitions run replicated on every rank (they are ~3 % of a level at C3, DESIGN.md §6).
"""
import json
import os
import time

import numpy as np

ITERATIONS = 10
GRID_LEVELS, RGBD_LEVELS = 3, 3
SHELL0, SHELL1 = 2.0, 1.0          # thin_shell_factor -> thin_shell_factor_final (data/intrinsic3d.yml)
LAM = dict(g=0.2, r0=80.0, r1=10.0, s0=120.0, s1=10.0, a=0.1)
OCCL, K = 0.02, 5


def _lerp(it, n, a, b):
    return a if n <= 1 else a + (b - a) * it / (n - 1)          # computeVaryingLambda (include/nv/refinement/cost.h:130-143)


def _pyramid(lum, depth, levels):
    """Pyramid stand-in (the reference builds it with cv::pyrDown / valid-average depth, out of scope): 2x2 mean luminance, subsampled depth."""
    out = [(lum, depth)]
    for _ in range(1, levels):
        l, d = out[-1]
        F, H, W = l.shape
        out.append((l.reshape(F, H // 2, 2, W // 2, 2).mean((2, 4)).astype(np.float32), np.ascontiguousarray(d[:, ::2, ::2])))
    return out


def run(args, rank, world, local_rank, dist, ClockSampler):
    import torch
    from intrinsic3d_b200 import engine
    from intrinsic3d_b200.ctypes_defs import default_params
    from intrinsic3d_b200.scene import make_color_frames, make_scene

    frames = int(os.environ.get("I3D_C5_FRAMES", "500"))
    s = make_scene(radius_vox=81.4, voxel_size=0.004, frames=frames, band=3.0, device=f"cuda:{local_rank}")
    col = make_color_frames(s)
    pyr = _pyramid(s["lum"], s["depth"], RGBD_LEVELS)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
    pyr = [(pin(l), pin(d)) for l, d in pyr]
    col = pin(col)
    n0 = len(s["xyz"])
    sdf0 = s["sdf0"].astype(np.float32).astype(np.float64)       # SDFAlgorithms::convert: the fused float sdf widened
    grid0 = dict(xyz=pin(s["xyz"]), sdf=pin(sdf0), alb=pin(np.full(n0, 0.6)), w=pin(s["weight"]), rgb=pin(s["rgb"]))
    F = frames

    eng = engine.Engine(local_rank)
    if world > 1:
        eng.comm_init(rank, world, dist)
    LP = engine.default_lighting_params()
    LP.subvolume_size = 0.2; LP.lambda_reg = 10.0; LP.weighted = 1
    stats = {}

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    def refine():
        """one Intrinsic3D::refine; returns (levels log, bytes host->device, bytes device->host)"""
        h2d = 0
        log = []
        eng.upload_grid(grid0["xyz"], grid0["sdf"], grid0["sdf"], grid0["alb"], grid0["w"], grid0["rgb"], s["voxel_size"])
        h2d += sum(v.nbytes for v in grid0.values()) + grid0["sdf"].nbytes
        eng.upload_frames(pyr[0][0], pyr[0][1], 1.0)
        eng.upload_color_frames(col)
        h2d += pyr[0][0].nbytes + pyr[0][1].nbytes + col.nbytes
        eng.set_camera(s["poses"], s["intr"], np.zeros(5))
        eng.recompute_colors(OCCL, K)
        vs = float(np.float32(s["voxel_size"]))
        level = 0
        for gl in range(GRID_LEVELS - 1, -1, -1):
            thres = _lerp(GRID_LEVELS - 1 - gl, GRID_LEVELS, SHELL0, SHELL1) * vs
            nvox = eng.clear_voxels_outside_thin_shell(thres)
            for rl in range(RGBD_LEVELS - 1, -1, -1):
                if rl > 0 and gl < GRID_LEVELS - 1:
                    continue
                t_lvl = time.perf_counter()
                if rl != level:
                    eng.upload_frames(pyr[rl][0], pyr[rl][1], 1.0 / 2 ** rl)
                    h2d += pyr[rl][0].nbytes + pyr[rl][1].nbytes
                    level = rl
                LP.thres_shell = thres
                li = eng.estimate_lighting(LP)
                if world > 1:
                    eng.set_shard(*engine.shard_range(nvox, rank, world))
                its = []
                for it in range(ITERATIONS):
                    p = default_params()
                    p.thres_shell = thres; p.occlusion_distance = OCCL; p.num_observations = K
                    p.lambda_[0] = LAM["g"]; p.lambda_[1] = _lerp(it, ITERATIONS, LAM["r0"], LAM["r1"])
                    p.lambda_[2] = _lerp(it, ITERATIONS, LAM["s0"], LAM["s1"]); p.lambda_[3] = LAM["a"]
                    info = eng.gn_iteration(p)
                    its.append((int(info.cg_iterations_total), int(info.step_accepted), float(info.cost_initial), float(info.cost_final)))
                if level != 0:
                    eng.upload_frames(pyr[0][0], pyr[0][1], 1.0)
                    eng.upload_color_frames(col)
                    h2d += pyr[0][0].nbytes + pyr[0][1].nbytes + col.nbytes
                    level = 0
                cnt = eng.recompute_colors(OCCL, K)
                torch.cuda.synchronize()
                log.append(dict(grid_level=gl, rgbd_level=rl, voxel_size=vs, voxels=int(nvox), active=int(info.num_active), eg_rows=int(info.type_residuals[0]),
                                subvolumes=int(li.num_subvolumes), cg_total=sum(x[0] for x in its), accepted=sum(x[1] for x in its),
                                cost_first=its[0][2], cost_last=its[-1][3], recolored=int(cnt[0]), wall_s=time.perf_counter() - t_lvl))
            if gl > 0:
                eng.upsample_grid()
                vs = float(np.float32(np.float32(vs) * np.float32(0.5)))
        g = eng.download_grid()
        st = eng.download_state()
        d2h = sum(v.nbytes for v in g.values() if hasattr(v, "nbytes")) + sum(v.nbytes for v in st.values())
        return log, h2d, d2h, {**g, **st}

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    refine()                                     # warm-up: allocations of the largest level, kernel attributes
    steps = max(1, args.steps)
    barrier()
    t0 = time.perf_counter()
    for _ in range(steps):
        log, h2d, d2h, outputs = refine()
    barrier()
    elapsed = time.perf_counter() - t0
    if dist is not None:
        t = torch.tensor([elapsed], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        elapsed = float(t.item())
    clocks = sampler.stop() if rank == 0 else None
    if rank == 0:
        gn = sum(ITERATIONS for _ in log)
        value = gn * steps / elapsed
        line = {"metric": "gauss_newton_iterations_per_sec", "value": value, "unit": "GN iter/s", "n_gpus": world, "steps": steps, "warmup": 1,
                "ms_per_step": 1e3 * elapsed / steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                "config": {"workload": "c5: coarse-to-fine 3-level refinement (0.5M -> 2M -> 8M voxels), %d frames 640x480, %d GN iterations per refinement" % (F, gn),
                           "voxels_level0": int(n0), "frames": int(F)},
                "parallelism": f"GN iterations voxel-sharded x{world}; lighting / recolouring / grid transitions replicated" if world > 1 else "single GPU",
                "step_definition": "one whole Intrinsic3D::refine through the C-ABI with host buffers (grid upload, frame uploads at level switches, pruning, lighting, 10 GN iterations per call, recolouring, upsampling, download)",
                "e2e": {"value": value, "unit": "GN iter/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h),
                        "note": "the whole schedule runs through the C-ABI with pinned host buffers: value IS the end-to-end number"},
                "clocks": clocks, "levels": log, "gn_iterations_per_step": gn}
        print(json.dumps(line))
    if dist is not None:
        dist.destroy_process_group()
    return outputs if rank == 0 else None
