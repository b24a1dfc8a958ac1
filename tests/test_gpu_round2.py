"""Round-2 GPU tests: parity on the configurations the numbers are quoted on (C2 whole, a C3 z-slab with all 200 frames),
camera state across frame re-uploads (pyramid-level switches of Intrinsic3D::refine), run-to-run bit-identity (small and full C3)."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _params(scene, **kw):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = scene["thres_shell"]
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _note(name, payload):
    """the achieved bounds, in the test's captured output (pytest -rA shows them); the tests never write into the tree"""
    print(f"test_{name}:", json.dumps(payload))


def test_camera_state_survives_frame_reupload(small_scene):
    """An accepted LM step swaps the engine's current/candidate camera buffers; re-uploading frames of the same count (what
    Intrinsic3D::refine does at every pyramid-level switch and before every recolouring) must keep the refined camera."""
    from intrinsic3d_b200.engine import Engine
    s = small_scene
    e = Engine(0)
    e.load_scene(s)
    p = _params(s)
    accepted = 0
    for it in range(3):
        info = e.gn_iteration(p)
        accepted += int(info.step_accepted)
        before = e.download_state()
        assert not np.allclose(before["poses"], s["poses"]) or accepted == 0
        e.upload_frames(s["lum"], s["depth"], 1.0)                 # same F, W, H
        after = e.download_state()
        for k in ("sdf_refined", "albedo", "poses", "intr", "dist"):
            assert np.array_equal(before[k], after[k]), (it, k)
        # a level switch: half-resolution frames, then back
        lum1 = s["lum"].reshape(s["lum"].shape[0], s["lum"].shape[1] // 2, 2, s["lum"].shape[2] // 2, 2).mean((2, 4)).astype(np.float32)
        e.upload_frames(lum1, np.ascontiguousarray(s["depth"][:, ::2, ::2]), 0.5)
        e.upload_frames(s["lum"], s["depth"], 1.0)
        after = e.download_state()
        for k in ("poses", "intr", "dist"):
            assert np.array_equal(before[k], after[k]), (it, k, "level switch")
    assert accepted >= 2          # odd and even numbers of buffer swaps were both exercised


def _lambda_ramp(p, it):
    """computeVaryingLambda (cost.h:130-143) over 10 iterations, yml defaults"""
    p.lambda_[1] = 80.0 - 70.0 / 9.0 * it
    p.lambda_[2] = 120.0 - 110.0 / 9.0 * it


def _info_bytes(info):
    """the bytes of every I3DIterInfo field before the wall-clock timers (time_add, time_build, time_solve come last)"""
    return bytes(info)[:type(info).time_add.offset]


def test_run_to_run_reproducibility(small_scene):
    """Two engines on identical inputs give bit-identical results: every float contribution of the iteration is summed in double,
    where the totals are exact and so independent of the order of the atomics, and rounded to float once."""
    from intrinsic3d_b200.engine import Engine
    s = small_scene
    outs, infos = [], []
    for _ in range(2):
        e = Engine(0)
        e.load_scene(s)
        p = _params(s)
        ii = []
        for it in range(3):
            _lambda_ramp(p, it)
            ii.append(e.gn_iteration(p))
        outs.append(e.download_state())
        infos.append(ii)
        e.close()
    moved = np.abs(outs[0]["sdf_refined"] - s["sdf_refined"]).max()
    cg = [[list(i.cg_iterations)[:i.lm_iterations] for i in ii] for ii in infos]
    _note("reproducibility", dict(scene="small", iterations=3, max_abs_sdf_update=float(moved), cg_iterations=cg))
    assert moved > 0
    for k in ("sdf_refined", "albedo", "poses", "intr", "dist"):
        assert outs[0][k].tobytes() == outs[1][k].tobytes(), k
    for a, b in zip(*infos):
        assert _info_bytes(a) == _info_bytes(b)


def test_c3_run_to_run_bit_identical():
    """The full C3 scene (2 M voxels, 200 frames; thousands of blocks add camera partials into the same double entries): two
    engines in turn, three GN iterations of the lambda ramp, byte-equal state and iteration info, then byte-equal b, s, jtj,
    cam_acc and one operator application."""
    import torch
    from intrinsic3d_b200.engine import Engine
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c3", device="cuda" if torch.cuda.is_available() else "cpu")
    engines = [Engine(0), Engine(0)]
    for e in engines:
        e.load_scene(s)
    p = _params(s)
    infos = [[], []]
    for it in range(3):
        _lambda_ramp(p, it)
        for i, e in enumerate(engines):
            infos[i].append(e.gn_iteration(p))
    for a, b in zip(*infos):
        assert _info_bytes(a) == _info_bytes(b)
    st = [e.download_state() for e in engines]
    for k in st[0]:
        assert st[0][k].tobytes() == st[1][k].tobytes(), k
    ne = [e.debug_normal_equations() for e in engines]
    for k in ne[0]:
        assert ne[0][k].tobytes() == ne[1][k].tobytes(), k
    U = 2 * engines[0].n + 6 * engines[0].F + 9
    v = np.random.default_rng(3).standard_normal(U).astype(np.float32)
    q = [e.debug_apply_operator(v) for e in engines]
    assert q[0].tobytes() == q[1].tobytes()
    n_active = int(infos[0][-1].num_active)
    _note("c3_reproducibility", dict(iterations=3, num_active=n_active, blocks_of_256=-(-n_active // 256),
                                     cg_iterations=[list(i.cg_iterations)[:i.lm_iterations] for i in infos[0]]))


def test_parity_c2_whole():
    """BASELINE config C2 (500 K voxels, 50 frames 640x480), the whole grid, one GN iteration against the oracle."""
    import torch
    from bench import parity_check
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c2", device="cuda" if torch.cuda.is_available() else "cpu")
    r = parity_check(s, 1.0, 0, min(32, os.cpu_count() or 8))
    _note("parity_c2", r)
    assert r["ok"], r
    assert r["residual_max_rel"] <= 1e-6 and r["eg_rows"] > 1_000_000


def test_parity_c3_slab():
    """BASELINE config C3 (2 M voxels, 200 frames): a 1/16 z-slab of the grid with ALL 200 frames against the oracle."""
    import torch
    from bench import parity_check
    from intrinsic3d_b200.scene import config_scene
    s = config_scene("c3", device="cuda" if torch.cuda.is_available() else "cpu")
    r = parity_check(s, 1.0 / 16.0, 0, min(32, os.cpu_count() or 8))
    _note("parity_c3_slab", r)
    assert r["ok"], r
    assert r["residual_max_rel"] <= 1e-6
