"""The cooperative k_cg_step (operator finish + PCG update + next direction in one grid) against the four-kernel chain it replaces
(I3D_PCG_FUSED=0): the same inputs give the same CG counts, LM trials and accept decisions and bit-equal x, p and step, and the fused
path is bit-identical from run to run."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# forced counts 1 / 2 / 21 (21 crosses the refresh iterations 10 and 20), and refresh period 3 (a fused iteration followed by a
# refresh iteration), with the adaptive Q-based stop too
CONFIGS = {
    "forced1": dict(forced_cg_iterations=1),
    "forced2": dict(forced_cg_iterations=2),
    "forced21": dict(forced_cg_iterations=21),
    "forced21_period3": dict(forced_cg_iterations=21, residual_reset_period=3),
    "adaptive": dict(),
    "adaptive_period3": dict(residual_reset_period=3),
}
_SCENES = {}


def _scene(name):
    if name not in _SCENES:
        import torch
        from intrinsic3d_b200.scene import config_scene
        _SCENES[name] = config_scene(name, device="cuda" if torch.cuda.is_available() else "cpu")
    return _SCENES[name]


def _engine(scene, fused):
    from intrinsic3d_b200.engine import Engine
    old = os.environ.get("I3D_PCG_FUSED")
    os.environ["I3D_PCG_FUSED"] = "1" if fused else "0"          # read when the engine is created
    try:
        e = Engine(0)
    finally:
        if old is None:
            del os.environ["I3D_PCG_FUSED"]
        else:
            os.environ["I3D_PCG_FUSED"] = old
    e.load_scene(scene)
    return e


def _info_bytes(info):
    """the bytes of every I3DIterInfo field before the wall-clock timers"""
    return bytes(info)[:type(info).time_add.offset]


def _decisions(info):
    lm = info.lm_iterations
    return lm, list(info.cg_iterations)[:lm], info.step_accepted, info.cg_iterations_total


@pytest.mark.parametrize("scene_name", ["tiny", "small", "c2"])
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_fused_step_matches_unfused_chain(scene_name, config):
    from intrinsic3d_b200.ctypes_defs import default_params
    s = _scene(scene_name)
    p = default_params()
    p.thres_shell = s["thres_shell"]
    for k, v in CONFIGS[config].items():
        setattr(p, k, v)
    fused, fused2, chain = _engine(s, True), _engine(s, True), _engine(s, False)
    report = []
    for it in range(3):
        p.lambda_[1] = 80.0 - 70.0 / 9.0 * it
        p.lambda_[2] = 120.0 - 110.0 / 9.0 * it
        a, a2, b = fused.gn_iteration(p), fused2.gn_iteration(p), chain.gn_iteration(p)
        assert _decisions(a) == _decisions(b), (it, _decisions(a), _decisions(b))
        assert _info_bytes(a) == _info_bytes(a2), it
        xa, pa = fused.debug_pcg_vectors()
        xa2, pa2 = fused2.debug_pcg_vectors()
        xb, pb = chain.debug_pcg_vectors()
        da, db = fused.debug_step()[0], chain.debug_step()[0]
        assert xa.tobytes() == xa2.tobytes() and pa.tobytes() == pa2.tobytes(), it
        assert da.tobytes() == fused2.debug_step()[0].tobytes(), it
        row = {"it": it, "cg": _decisions(b)[1]}
        for vec, va, vb in (("x", xa, xb), ("p", pa, pb), ("step", da, db)):
            row[vec + "_entries_differing"] = int(np.count_nonzero(va.view(np.uint8) != vb.view(np.uint8)))
        # every float expression per unknown is the chain's, rounded the same way: the iterates are bit-equal
        assert xa.tobytes() == xb.tobytes() and pa.tobytes() == pb.tobytes() and da.tobytes() == db.tobytes(), row
        report.append(row)
        sa, sa2, sb = fused.download_state(), fused2.download_state(), chain.download_state()
        for k in sa:
            assert sa[k].tobytes() == sa2[k].tobytes(), (it, k)
        # the next iteration starts from identical inputs on all three engines
        for e in (fused, fused2, chain):
            e.upload_voxel_params(sb["sdf_refined"], sb["albedo"])
            e.set_camera(sb["poses"], sb["intr"], sb["dist"])
    for e in (fused, fused2, chain):
        e.close()
    print(f"test_pcg_step[{scene_name}-{config}]:", json.dumps(report))
