"""The launch count of a GN iteration (phase "launches", the bench's gpu_launches) against the kernels the device actually ran: for
each case, phase_count("launches") equals the number of engine kernels (namespace i3d) torch.profiler records during the one
gn_iteration call, so the count neither misses a launch nor counts one that was skipped."""
import json
import os
import re

import pytest

pytestmark = pytest.mark.gpu

CASES = {
    "fused": (True, {}),
    "chain": (False, {}),
    # refresh period 3 with 4 forced PCG iterations: iteration 3 is a refresh (operator applied twice, the chain's kernels on the
    # fused path too)
    "refresh": (True, dict(residual_reset_period=3, forced_cg_iterations=4)),
    # no voxel lies within a negative shell: k_flags marks no row, and every kernel that needs rows is skipped
    "no_rows": (True, dict(thres_shell=-1.0)),
}
_SCENES = {}


def _scene():
    if "small" not in _SCENES:
        from intrinsic3d_b200.scene import config_scene
        _SCENES["small"] = config_scene("small", device="cuda")
    return _SCENES["small"]


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


def _is_engine_kernel(ev):
    import torch
    return ev.device_type == torch.autograd.DeviceType.CUDA and re.match(r"(void )?i3d::|_ZN3i3d", ev.name) is not None


@pytest.mark.parametrize("case", sorted(CASES))
def test_launch_count_matches_profiled_kernels(case):
    import torch
    from intrinsic3d_b200.ctypes_defs import default_params
    fused, over = CASES[case]
    s = _scene()
    p = default_params()
    p.thres_shell = s["thres_shell"]
    for k, v in over.items():
        setattr(p, k, v)
    e = _engine(s, fused)
    try:
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            info = e.gn_iteration(p)
        counted = e.phase_count("launches")
    finally:
        e.close()
    kernels = [ev.name.split("(")[0] for ev in prof.events() if _is_engine_kernel(ev)]
    by_name = {}
    for k in kernels:
        by_name[k] = by_name.get(k, 0) + 1
    print(f"test_launch_count[{case}]:", json.dumps(dict(num_active=int(info.num_active), counted=counted, profiled=len(kernels),
                                                         kernels=by_name)))
    if case == "no_rows":
        assert info.num_active == 0
    else:
        assert info.num_active > 0
    if case == "refresh":
        assert any("k_x_update" in k for k in kernels), by_name
    assert counted == len(kernels), by_name
