"""The device Levenberg-Marquardt trial against the float64 restatement of tests/lm_trial_ref.py, built from the engine's own rows,
gradient, Jacobi scale, diagonal and camera sums of the same iteration, so that what is measured is the solve kernels' arithmetic:

  A  step delta.  After one PCG iteration componentwise, |gpu - ref|_j <= c_j 2^-24 M_j (lm_trial_ref.k1_bound derives c_j);
     after k >= 2 per block [sdf | albedo | poses | intr | dist]:  ||gpu - ref||_inf <= 8 max_e ||emu_e - ref||_inf + 2^-20 ||ref||_inf
     over two float32 emulations of the same recurrence (lm_trial_ref.pcg(f32=True)): one with the operator product rounded once,
     one with the engine's own operator kernels (Engine.debug_apply_operator, pinned entry by entry by test_gpu_normal_equations.py).
     The second is needed: the operator's float sums are the dominant error of the ill-conditioned 5 x 5 distortion block, and the
     once-rounded emulation's error there is a single draw that varied 16x between two trials of the same run (measured on an H100:
     trial 2 of a two-trial rejection, engine 4.9e-4 from ref, once-rounded emulation 3.1e-5, engine-operator emulation 6.1e-4).
     Fixed unknowns and frames no row sees must be exactly 0, and fixed unknowns keep their bytes.
  B  model cost change 0.5 (x.D^2 x - Q1) from the PCG scalars against the explicit -sum w m (f + m/2) at the engine's own delta,
     bound 8 max_e |emu_e scalar - explicit(delta_e)| (the residual drift) + the rounding terms of
     lm_trial_ref.model_cost_change_bound
  C  the candidate: an accepted state equals state0 + float64(delta) byte for byte, a rejected one keeps its bytes; the candidate
     cost equals the restatement at state0 + float64(delta) on the frozen rows to rel 1e-11
  D  C at F = 479 (pose table staged in shared memory) and F = 480 (read through L1) by k_eg_rows<ROWS_COST>
  E  every exit of the trial loop, driven by parameters: engine and oracle agree on trials, termination, acceptance and CG counts;
     the engine's radius equals the restated k_lm_decide on its own reported costs bit for bit
  F  the PCG iteration count carried from solve to solve
Every test prints its achieved error-to-bound ratios (pytest -rA shows them).
"""
import json
import os
import re

import numpy as np
import pytest

import lm_trial_ref as ltr
import normal_equations_ref as ner

pytestmark = pytest.mark.gpu

# k_eg_rows<ROWS_COST> stages the F x 176 B pose table while 2 (128 + ceil_128(176 F) + 256 * 15 * 8 + 1024) <= 227 KB
# (launch_eg_rows; sizeof(FramePose) == 176 is a static_assert in i3d_math.cuh)
STAGE_MAX_F = max(F for F in range(1, 2000) if 2 * (128 + ((176 * F + 127) // 128) * 128 + 256 * 15 * 8 + 1024) <= 227 * 1024)


def _params(scene, **kw):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = scene["thres_shell"]
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _copy(p):
    return type(p).from_buffer_copy(bytes(p))


def _note(name, payload):
    print(f"test_{name}:", json.dumps(payload))


def _state(scene):
    return dict(sdf_refined=np.asarray(scene["sdf_refined"], np.float64).copy(), albedo=np.asarray(scene["albedo"], np.float64).copy(),
                poses=np.asarray(scene["poses"], np.float64).copy(), intr=np.asarray(scene["intr"], np.float64).copy(),
                dist=np.asarray(scene["dist"], np.float64).copy())


def invalid_black_scene(tiny):
    """the scene of test_invalid_and_black_voxels: weight-0 and black voxels, distortion, a coarser pyramid level"""
    s = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in tiny.items()}
    rng = np.random.default_rng(7)
    n = s["xyz"].shape[0]
    s["weight"][rng.choice(n, n // 50, replace=False)] = 0.0
    s["rgb"][rng.choice(n, n // 40, replace=False)] = 0
    s["dist"] = np.array([0.02, -0.01, 0.003, 0.001, -0.0007])
    s["intr"] = s["intr"] * 2.0
    s["pyr_scale"] = 0.5
    return s


def run_engine(e, scene, p):
    """one engine iteration and everything the restatement needs from it"""
    from oracle import Oracle
    state0 = e.download_state()
    info = e.gn_iteration(_copy(p))
    host_syncs = e.phase_count("host_syncs")
    rows = e.debug_rows()
    ne = e.debug_normal_equations()
    delta = e.debug_step()[0]
    state1 = e.download_state()
    tw = np.array(list(info.type_weights))
    sl = np.nonzero(rows["frame"] >= 0)[0]
    eg = dict(voxel=rows["voxel"][sl], frame=rows["frame"][sl], residual=rows["residual"][sl], raw_weight=rows["raw_weight"][sl],
              J=rows["J"][:, sl].T.astype(np.float64), w_op=np.float32(rows["raw_weight"][sl] * tw[0]).astype(np.float64))
    s0 = dict(scene)
    s0.update(state0)
    o = Oracle(threads=min(32, os.cpu_count() or 8))
    o.load_scene(s0)
    pb = _copy(p)
    pb.build_only = 1
    o.gn_iteration(pb)
    reg = (o.rows(1), o.rows(2), o.rows(3))
    R = ner.build_rows(s0, eg, reg, tw)
    S = ltr.System(R, ne["s"], ne["b"], ne["jtj"], ne["cam_acc"], tw[0])
    K = p.num_observations if 0 < p.num_observations <= R.F else R.F
    return dict(info=info, eg=eg, reg=reg, tw=tw, R=R, S=S, ne=ne, delta=delta, state0=state0, state1=state1, scene=s0,
                free=ne["s"] != 0, e=e, K=K, host_syncs=host_syncs)


def decision_chain(r, p):
    """the restated k_lm_decide over the engine's reported costs: per trial (radius it ran with, decision)"""
    info = r["info"]
    radius, df = p.initial_trust_region_radius, 2.0
    x = np.concatenate([r["state0"][k].ravel() for k in ("sdf_refined", "albedo", "poses", "intr", "dist")])
    xn = float(np.sqrt(np.sum(x[r["free"] & (r["ne"]["jtj"] > 0)] ** 2)))
    out = []
    for t in range(info.lm_iterations):
        # only the last trial's step norm is reported; earlier trials were decided on rho, far above the parameter tolerance
        sn = info.step_norm if t == info.lm_iterations - 1 else 1.0
        dec = ltr.lm_decide(info.cost_initial, info.model_cost_change[t], info.candidate_cost[t], sn, xn, radius, df, t + 1, p)
        out.append((radius, dec))
        radius, df = dec["radius"], dec["decrease_factor"]
    return out


def check_trial(r, p, name):
    """A, B and C for the last trial of the iteration, asserted; prints and returns the achieved ratios"""
    info, R, S, e = r["info"], r["R"], r["S"], r["e"]
    chain = decision_chain(r, p)
    last = info.lm_iterations - 1
    radius = chain[-1][0]
    ref = ltr.pcg(S, p, radius)
    emus = [ltr.pcg(S, p, radius, f32=True), ltr.pcg(S, p, radius, f32=True, apply_op=lambda v: e.debug_apply_operator(np.float32(v)))]
    delta = np.asarray(r["delta"], np.float64)
    res = {}
    # A: step
    step = ltr.block_compare(delta, [m["delta"] for m in emus], ref["delta"], R.n, R.F)
    res["step"] = step
    if info.cg_iterations[last] == 1:
        ref1, bnd = ltr.k1_bound(S, p, radius)
        err = np.abs(delta - ref1)
        assert np.all(err[bnd == 0] == 0)
        res["step_k1_componentwise"] = float(np.max(err[bnd > 0] / bnd[bnd > 0]))
    free = r["free"]
    assert np.all(delta[~free] == 0)
    x0 = np.concatenate([r["state0"][k].ravel() for k in ("sdf_refined", "albedo", "poses", "intr", "dist")])
    x1 = np.concatenate([r["state1"][k].ravel() for k in ("sdf_refined", "albedo", "poses", "intr", "dist")])
    assert x1[~free].tobytes() == x0[~free].tobytes()
    seen = np.bincount(r["eg"]["frame"], minlength=R.F) > 0
    assert np.all(delta[2 * R.n:2 * R.n + 6 * R.F].reshape(R.F, 6)[~seen] == 0)
    # CG count: equal to the float64 restatement's, or one off where eta lies between the zeta of the float64 and the float32
    # recurrences at the iteration where one stopped and the other did not (widened by 1e-6 eta): the stop is then decided by
    # rounding.  (A 40-iteration solve at eta 1e-3 moves zeta by far more than 1e-6 of eta between float32 and float64.)
    cg = info.cg_iterations[last]
    if cg != ref["it"]:
        i = min(cg, ref["it"])
        z = [m["zetas"][i - 1] for m in [ref] + emus if len(m["zetas"]) >= i]
        ok = p.forced_cg_iterations == 0 and abs(cg - ref["it"]) == 1 and min(z) - 1e-6 * p.eta <= p.eta <= max(z) + 1e-6 * p.eta
        print(f"test_{name}: CG count {cg} vs restated {ref['it']}, zeta at iteration {i}: {z}, eta {p.eta}")
        assert ok, (cg, ref["it"], z)
    # B: model cost change
    x = np.where(S.s != 0, -delta / np.where(S.s != 0, S.s, 1.0), 0.0)
    drift = max(abs(0.5 * (m["xd2x"] - m["Q1"]) - ltr.model_cost_change(R, m["delta"])) for m in emus)
    bound = 8 * drift + ltr.model_cost_change_bound(R, S, x, delta, r["K"], S.d2(p, radius))
    res["model_cost_change"] = abs(info.model_cost_change[last] - ltr.model_cost_change(R, delta)) / bound
    # C: candidate
    cand_state = ltr.apply_step(r["state0"], delta, R.n, R.F)
    accepted = bool(info.step_accepted)
    for k in r["state1"]:
        want = cand_state[k] if accepted else r["state0"][k]
        assert r["state1"][k].tobytes() == want.tobytes(), (k, accepted)
    if info.candidate_cost[last] != 0:          # recorded for every valid step
        ea_w = np.float32(r["reg"][2]["raw_weight"]).astype(np.float64)
        cand = ltr.candidate_cost(r["scene"], cand_state, r["eg"], r["reg"], ea_w, r["tw"])[0]
        res["candidate_rel"] = abs(info.candidate_cost[last] - cand) / abs(cand)
        assert res["candidate_rel"] <= 1e-11, res
    # E: the radius bit for bit
    assert info.trust_region_radius == chain[-1][1]["radius"], (info.trust_region_radius, chain[-1][1]["radius"])
    _note(name, dict(trials=info.lm_iterations, cg=list(info.cg_iterations[:info.lm_iterations]), restated_cg=ref["it"],
                     max_err_over_bound=res))
    assert max(step.values()) <= 1.0, step
    assert res.get("step_k1_componentwise", 0.0) <= 1.0, res
    assert res["model_cost_change"] <= 1.0, res
    return res


def away_frame_scene(tiny):
    """the tiny scene plus one frame 100 units behind the first camera: no row sees it, so its pose block is zero"""
    s = dict(tiny)
    pose = s["poses"][:1].copy()
    pose[0, 3:] += np.array([0.0, 0.0, -100.0])
    s["poses"] = np.concatenate([s["poses"], pose])
    s["lum"] = np.concatenate([s["lum"], s["lum"][:1]])
    s["depth"] = np.concatenate([s["depth"], s["depth"][:1]])
    return s


def _engine(scene):
    from intrinsic3d_b200.engine import Engine
    e = Engine(0)
    e.load_scene(scene)
    return e


# ---- A / B / C ------------------------------------------------------------------------------------------------------------------
STEP_CASES = [("small", dict(forced_cg_iterations=k)) for k in (1, 2, 9, 10, 11, 21)] + [
    ("tiny", dict(forced_cg_iterations=10, residual_reset_period=1)),
    ("tiny", dict(forced_cg_iterations=10, residual_reset_period=3)),
    ("tiny", dict(forced_cg_iterations=11, initial_trust_region_radius=1e-3)),
    ("tiny", dict(forced_cg_iterations=11, initial_trust_region_radius=1e4)),
    ("tiny", dict(forced_cg_iterations=11, initial_trust_region_radius=1e12)),
    ("tiny", dict(forced_cg_iterations=9, max_lm_diagonal=1e-4)),
    ("invalid_black", dict(forced_cg_iterations=10, num_observations=8)),
    ("tiny", dict(forced_cg_iterations=10, fix_poses=1)),
    ("tiny", dict(forced_cg_iterations=10, fix_intrinsics=1, fix_distortion=1)),
    ("away_frame", dict(forced_cg_iterations=10)),
    ("tiny", {}),
]


@pytest.mark.parametrize("case", STEP_CASES, ids=lambda c: c[0] + "_" + "_".join(f"{k}{v}" for k, v in c[1].items()))
def test_trial_against_restatement(case, tiny_scene, small_scene):
    name, kw = case
    s = dict(tiny=tiny_scene, small=small_scene, invalid_black=None, away_frame=None)[name]
    if name == "invalid_black":
        s = invalid_black_scene(tiny_scene)
    if name == "away_frame":
        s = away_frame_scene(tiny_scene)
    p = _params(s, **kw)
    if "max_lm_diagonal" in kw:
        e = _engine(s)
        r = run_engine(e, s, p)
        assert np.mean(r["ne"]["jtj"][r["free"]] > kw["max_lm_diagonal"]) > 0.5       # the clamp is active on most unknowns
    else:
        r = run_engine(_engine(s), s, p)
    if name == "away_frame":
        assert not np.any(r["eg"]["frame"] == r["R"].F - 1)          # the frame no row sees
    cam_free = r["free"][2 * r["R"].n:]
    if kw.get("fix_poses"):
        assert not np.any(cam_free[:-9])
    if kw.get("fix_intrinsics"):
        assert not np.any(cam_free[-9:-5]) and not np.any(cam_free[-5:])
    check_trial(r, p, f"trial[{name}_{kw}]")


@pytest.mark.parametrize("F", [STAGE_MAX_F, STAGE_MAX_F + 1])
def test_cost_staging_boundary(F):
    """D: the candidate cost on both sides of the pose-table staging limit of k_eg_rows<ROWS_COST>"""
    from intrinsic3d_b200.scene import config_scene
    import torch
    assert STAGE_MAX_F == 479
    assert os.environ.get("I3D_ROWS_STAGE", "1") == "1", "I3D_ROWS_STAGE forces one k_eg_rows variant"
    s = config_scene("tiny", frames=F, width=32, height=24)
    p = _params(s, num_observations=5, forced_cg_iterations=3)
    e = _engine(s)
    # which k_eg_rows<ROWS_COST = 1, THREADS, STAGE> instance ran, from the kernel names the profiler records
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        r = run_engine(e, s, p)
    names = {ev.name for ev in prof.events() if "k_eg_rows" in ev.name}
    cost = [n for n in names if re.search(r"k_eg_rows<\(?int\)?1, ", n) or re.search(r"k_eg_rows<1,", n)]
    _note(f"staging_variant[F{F}]", sorted(names))
    assert cost, sorted(names)
    want = "256, true" if F <= STAGE_MAX_F else "128, false"
    assert all(want in n.replace("(int)", "").replace("(bool)", "") for n in cost), (F, cost)
    check_trial(r, p, f"staging[F{F}]")


# ---- E: the exits of the trial loop -----------------------------------------------------------------------------------------
EXITS = {
    "accept": {},
    "reject_lm1": dict(min_relative_decrease=2.0, lm_steps=1),
    "reject_lm2": dict(min_relative_decrease=2.0, lm_steps=2),
    "reject_lm4": dict(min_relative_decrease=2.0, lm_steps=4),
    "min_radius": dict(min_relative_decrease=2.0, min_trust_region_radius=1e4 / 8 * 1.5),
    "max_radius": dict(max_trust_region_radius=5e3),
    "function_tolerance": dict(function_tolerance=1.0),
    "parameter_tolerance": dict(parameter_tolerance=1e30),
}


def _oracle_iteration(scene, p):
    from oracle import Oracle
    o = Oracle(threads=min(32, os.cpu_count() or 8))
    o.load_scene(scene)
    return o.gn_iteration(_copy(p))


def _agree(ie, io):
    n = io.lm_iterations
    assert (ie.lm_iterations, ie.termination, ie.step_accepted) == (io.lm_iterations, io.termination, io.step_accepted), \
        ((ie.lm_iterations, ie.termination, ie.step_accepted), (io.lm_iterations, io.termination, io.step_accepted))
    assert all(abs(a - b) <= 1 for a, b in zip(ie.cg_iterations[:n], io.cg_iterations[:n])), (list(ie.cg_iterations[:n]), list(io.cg_iterations[:n]))


@pytest.mark.parametrize("name", list(EXITS))
def test_exit(name, tiny_scene):
    s = tiny_scene
    p = _params(s, **EXITS[name])
    r = run_engine(_engine(s), s, p)
    io = _oracle_iteration(s, p)
    ie = r["info"]
    _agree(ie, io)
    if name.startswith("reject"):
        k = EXITS[name]["lm_steps"]
        assert all(ie.relative_decrease[t] < 2.0 for t in range(k))
        assert ie.trust_region_radius == 1e4 / 2.0 ** (k * (k + 1) // 2)
    if name == "min_radius":
        assert ie.lm_iterations == 2 and ie.termination == 1
    if name == "max_radius":
        assert ie.step_accepted and ie.trust_region_radius == 5e3
    if name in ("function_tolerance", "parameter_tolerance"):
        assert ie.termination == 1 and not ie.step_accepted
    check_trial(r, p, f"exit[{name}]")


def test_reject_then_accept(tiny_scene):
    s = tiny_scene
    base = dict(initial_trust_region_radius=1.0)
    io = _oracle_iteration(s, _params(s, min_relative_decrease=2.0, lm_steps=2, **base))
    rho1, rho2 = io.relative_decrease[0], io.relative_decrease[1]
    assert rho1 < rho2
    p = _params(s, min_relative_decrease=0.5 * (rho1 + rho2), **base)
    r = run_engine(_engine(s), s, p)
    ie = r["info"]
    assert ie.relative_decrease[0] < p.min_relative_decrease < ie.relative_decrease[1]
    _agree(ie, _oracle_iteration(s, p))
    assert ie.lm_iterations == 2 and ie.step_accepted
    check_trial(r, p, "reject_then_accept")


def _gradient_norms(scene, p):
    """(max-norm, 2-norm) of the unscaled gradient over the free unknowns, from the oracle's rows"""
    import test_lm_trial_ref as tref
    R, _, _, _, _ = tref.oracle_problem(scene, p)
    c = tref.oracle_case(scene, p)
    return ltr.gradient_norms(R, c["free"])


@pytest.mark.parametrize("where", ["between", "above_max", "below_max"])
def test_gradient_tolerance(where, tiny_scene):
    """Ceres tests the max-norm of the unscaled gradient: a tolerance between the max-norm and the 2-norm stops both with 0 trials"""
    s = tiny_scene
    gmax, g2 = _gradient_norms(s, _params(s))
    tol = dict(between=np.sqrt(gmax * g2), above_max=gmax * 1.01, below_max=gmax * 0.99)[where]
    p = _params(s, gradient_tolerance=tol)
    ie = _engine(s).gn_iteration(_copy(p))
    io = _oracle_iteration(s, p)
    _note(f"gradient_tolerance[{where}]", dict(gmax=gmax, g2=g2, tol=tol, engine=(ie.termination, ie.lm_iterations),
                                                oracle=(io.termination, io.lm_iterations)))
    stops = where != "below_max"
    assert (io.termination == 1 and io.lm_iterations == 0) == stops
    _agree(ie, io)


def test_preconditioner_not_spd(tiny_scene):
    """min_lm_diagonal = max_lm_diagonal = 0 and one extra frame no row sees: its pose block is zero, termination 3, state kept"""
    s = away_frame_scene(tiny_scene)
    p = _params(s, min_lm_diagonal=0.0, max_lm_diagonal=0.0)
    e = _engine(s)
    st0 = e.download_state()
    ie = e.gn_iteration(_copy(p))
    rows = e.debug_rows(want_jac=False)
    assert not np.any(rows["frame"] == s["poses"].shape[0] - 1)
    io = _oracle_iteration(s, p)
    assert ie.termination == 3 and io.termination == 3 and not ie.step_accepted
    st1 = e.download_state()
    for k in st0:
        assert st0[k].tobytes() == st1[k].tobytes(), k


# ---- F: PCG count carry-over ----------------------------------------------------------------------------------------------------
def test_cg_count_carry_over(small_scene):
    """eta 0.1, then 1e-3 (the host enqueues fewer iterations than the solve needs and adds two at a time), then 0.5 (more than
    needed: the extra iterations must be no-ops)"""
    s = dict(small_scene)
    e = _engine(s)
    counts, syncs = [], []
    for i, eta in enumerate((0.1, 1e-3, 0.5)):
        p = _params(s, eta=eta)
        r = run_engine(e, s, p)
        check_trial(r, p, f"carry_over[{i}_eta{eta}]")
        assert r["info"].lm_iterations == 1
        counts.append(r["info"].cg_iterations[0])
        syncs.append(r["host_syncs"])
        s.update(r["state1"])
    _note("carry_over_batches", dict(cg=counts, host_syncs=syncs))
    # one sync after the activity scan + one per decision round; the first round enqueues max(last two solves) iterations (the
    # engine starts from 4 and 4)
    first = max(counts[0], 4)
    assert counts[1] > first and syncs[1] == 2 + -(-(counts[1] - first) // 2)                # fewer enqueued than needed: 2 at a time
    assert counts[2] < max(counts[:2]) and syncs[2] == 2                                      # more enqueued than needed: no-ops
