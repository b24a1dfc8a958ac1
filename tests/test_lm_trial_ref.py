"""tests/lm_trial_ref.py pinned to the oracle: fed the oracle's float64 rows, Jacobi scale and diagonal, the restatement reproduces
the oracle's step, model cost change, candidate cost, CG counts, radius and termination for every exit of the trial loop; and the
comparator's self-test: each deliberate error of lm_trial_ref.Perturb breaks the bounds the GPU test applies.  No GPU needed."""
import os

import numpy as np
import pytest

import lm_trial_ref as ltr
import normal_equations_ref as ner


def _params(scene, **kw):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = scene["thres_shell"]
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _copy(p):
    return type(p).from_buffer_copy(bytes(p))


def state_of(scene):
    return dict(sdf_refined=np.asarray(scene["sdf_refined"], np.float64), albedo=np.asarray(scene["albedo"], np.float64),
                poses=np.asarray(scene["poses"], np.float64), intr=np.asarray(scene["intr"], np.float64),
                dist=np.asarray(scene["dist"], np.float64))


def oracle_problem(scene, p):
    """(rows R with float64 operator weights, eg rows, regulariser rows, type weights, free mask, ref normal equations) from a
    build-only oracle iteration at the scene's state"""
    from oracle import Oracle
    o = Oracle(threads=min(16, os.cpu_count() or 4))
    o.load_scene(scene)
    pb = _copy(p)
    pb.build_only = 1
    info = o.gn_iteration(pb)
    tw = np.array(list(info.type_weights))
    r0 = o.rows(0)
    eg = dict(voxel=r0["voxel"], frame=r0["aux"], residual=r0["residual"], raw_weight=r0["raw_weight"], J=o.eg_jacobian(),
              w_op=r0["raw_weight"] * tw[0])
    reg = (o.rows(1), o.rows(2), o.rows(3))
    R = ner.build_rows(scene, eg, reg, tw)
    R.w_op = list(R.w)
    return R, eg, reg, tw, info


def oracle_case(scene, p):
    """the oracle's full iteration and the restatement of its trials from the oracle's own rows"""
    from oracle import Oracle
    R, eg, reg, tw, _ = oracle_problem(scene, p)
    o = Oracle(threads=min(16, os.cpu_count() or 4))
    o.load_scene(scene)
    info = o.gn_iteration(_copy(p))
    step, free, cs = o.step()
    free = free.astype(bool)
    ev = ner.evaluate(R, free, np.where(free, cs, 0.0))
    S = ltr.System(R, ev["s"][0], ev["b"][0], ev["jtj"][0], ev["cam_acc"][0], tw[0])
    return dict(R=R, eg=eg, reg=reg, tw=tw, info=info, step=step, free=free, S=S, state=state_of(scene), o=o)


def x_norm(state, free, colnorm_pos):
    x = np.concatenate([state["sdf_refined"], state["albedo"], state["poses"].ravel(), state["intr"], state["dist"]])
    m = free & colnorm_pos
    return float(np.sqrt(np.sum(x[m] ** 2)))


def restate_trials(c, scene, p, ea_w=None, fma=False, perturb=None):
    """Every trial of the oracle's loop restated.  The decision chain is driven by the oracle's reported costs (so the radius can be
    compared bit for bit); the restated CG counts, model cost change and candidate cost are returned per trial for comparison."""
    info, S, R = c["info"], c["S"], c["R"]
    ea_w = c["reg"][2]["raw_weight"] if ea_w is None else ea_w
    radius, df = p.initial_trust_region_radius, 2.0
    trials = []
    for t in range(info.lm_iterations):
        res = ltr.pcg(S, p, radius, perturb=perturb)
        tr = dict(radius=radius, pcg=res)
        if not res["ok"]:
            tr.update(termination=3)
            trials.append(tr)
            break
        d = res["delta"]
        tr["mcc"] = ltr.model_cost_change(R, d)
        tr["cand"] = ltr.candidate_cost(scene, ltr.apply_step(c["state"], d, R.n, R.F), c["eg"], c["reg"], ea_w, c["tw"], perturb)[0]
        dec = ltr.lm_decide(info.cost_initial, info.model_cost_change[t], info.candidate_cost[t], info.step_norm if t == info.lm_iterations - 1
                            else np.sqrt(np.sum(d * d)), x_norm(c["state"], c["free"], S.jtj > 0), radius, df, t + 1, p, fma=fma)
        tr["decision"] = dec
        trials.append(tr)
        radius, df = dec["radius"], dec["decrease_factor"]
        if dec["state"] != "running":
            break
    return trials


def check_against_oracle(c, trials, p):
    info, R = c["info"], c["R"]
    assert len(trials) == info.lm_iterations
    for t, tr in enumerate(trials):
        assert tr["pcg"]["it"] == info.cg_iterations[t], (t, tr["pcg"]["it"], info.cg_iterations[t])
        if "mcc" in tr:
            assert abs(tr["mcc"] - info.model_cost_change[t]) <= 1e-10 * abs(info.model_cost_change[t]), (t, tr["mcc"], info.model_cost_change[t])
            assert abs(tr["cand"] - info.candidate_cost[t]) <= 1e-12 * abs(info.candidate_cost[t]), (t, tr["cand"], info.candidate_cost[t])
    last = trials[-1]
    if last["pcg"]["ok"]:
        for k, sl in ltr.blocks(R.n, R.F).items():
            ref, got = c["step"][sl], last["pcg"]["delta"][sl]
            scale = np.abs(ref).max() if ref.size else 0.0
            assert np.abs(got - ref).max() <= 1e-10 * scale if scale > 0 else np.all(got == 0), k
        dec = last["decision"]
        assert dec["termination"] == info.termination
        assert dec["radius"] == info.trust_region_radius, (dec["radius"], info.trust_region_radius)
        assert int(dec["accepted"]) == info.step_accepted
    else:
        assert info.termination == 3 and last["termination"] == 3


# the exits of the trial loop, driven by parameters only (the same cases as tests/test_gpu_lm_trial.py)
EXITS = {
    "accept": {},
    "reject_lm1": dict(min_relative_decrease=2.0, lm_steps=1),
    "reject_lm2": dict(min_relative_decrease=2.0, lm_steps=2),
    "reject_lm4": dict(min_relative_decrease=2.0, lm_steps=4),
    "min_radius": dict(min_relative_decrease=2.0, min_trust_region_radius=1e4 / 8 * 1.5),
    "max_radius": dict(max_trust_region_radius=5e3),
    "function_tolerance": dict(function_tolerance=1.0),
    "parameter_tolerance": dict(parameter_tolerance=1e30),
    "forced_k10_reset3": dict(forced_cg_iterations=10, residual_reset_period=3),
    "radius_1e-3": dict(initial_trust_region_radius=1e-3, forced_cg_iterations=11),
    "clamp_active": dict(max_lm_diagonal=1e-4, forced_cg_iterations=9),
}


@pytest.mark.parametrize("name", list(EXITS))
def test_restatement_reproduces_oracle(name, tiny_scene):
    s = tiny_scene
    p = _params(s, **EXITS[name])
    c = oracle_case(s, p)
    trials = restate_trials(c, s, p)
    if name.startswith("reject_lm"):
        k = EXITS[name]["lm_steps"]
        assert c["info"].lm_iterations == k and c["info"].step_accepted == 0
        assert c["info"].trust_region_radius == 1e4 / 2.0 ** (k * (k + 1) // 2)
    if name == "min_radius":
        assert c["info"].lm_iterations == 2 and c["info"].termination == 1
    check_against_oracle(c, trials, p)


REJECT_THEN_ACCEPT = dict(initial_trust_region_radius=1.0)


def test_reject_then_accept(tiny_scene):
    """threshold between the first two trials' relative decrease (taken from an oracle run at lm_steps = 2, threshold 2); at the
    initial radius 1 the halved radius gives the larger relative decrease"""
    s = tiny_scene
    c0 = oracle_case(s, _params(s, min_relative_decrease=2.0, lm_steps=2, **REJECT_THEN_ACCEPT))
    rho1, rho2 = c0["info"].relative_decrease[0], c0["info"].relative_decrease[1]
    assert rho1 < rho2, (rho1, rho2)
    p = _params(s, min_relative_decrease=0.5 * (rho1 + rho2), **REJECT_THEN_ACCEPT)
    c = oracle_case(s, p)
    assert c["info"].lm_iterations == 2 and c["info"].step_accepted == 1
    check_against_oracle(c, restate_trials(c, s, p), p)


def test_gradient_tolerance_between_the_norms(tiny_scene):
    """the oracle stops on the max-norm of the unscaled gradient; a tolerance between max-norm and 2-norm stops it with 0 trials"""
    s = tiny_scene
    R, _, _, _, _ = oracle_problem(s, _params(s))
    c = oracle_case(s, _params(s))
    gmax, g2 = ltr.gradient_norms(R, c["free"])
    assert gmax < g2
    for tol, stops in ((np.sqrt(gmax * g2), True), (gmax * 1.01, True), (gmax * 0.99, False)):
        from oracle import Oracle
        o = Oracle(threads=4)
        o.load_scene(s)
        info = o.gn_iteration(_params(s, gradient_tolerance=tol))
        assert (info.termination == 1 and info.lm_iterations == 0) == stops, (tol, info.termination, info.lm_iterations)


# ---- the comparator's own test ------------------------------------------------------------------------------------------------
def _perturbed_ratio(c, p, perturb, radius):
    """max over blocks of ||delta_pert - delta_ref|| / (8 max_e ||delta_emu_e - delta_ref|| + 2^-20 ||delta_ref||), the emulations
    being the once-rounded one and, standing in for the engine's operator kernels of the GPU test, one whose operator products carry
    random errors of the full size test_gpu_normal_equations allows them (rounding_counts(K)["q"] 2^-24 M)"""
    S, R = c["S"], c["R"]
    ref = ltr.pcg(S, p, radius)
    cq = ner.rounding_counts(p.num_observations)["q"]
    emus = [ltr.pcg(S, p, radius, f32=True)["delta"]] + [ltr.pcg(S, p, radius, f32=True, op_noise=(cq, seed))["delta"] for seed in (1, 2, 3)]
    bad = ltr.pcg(S, p, radius, perturb=perturb)
    return max(ltr.block_compare(bad["delta"], emus, ref["delta"], R.n, R.F).values())


@pytest.mark.parametrize("which", ["pose_offdiag", "radius_x2", "stale_refresh"])
def test_perturbation_breaks_step_bound(which, tiny_scene):
    s = tiny_scene
    p = _params(s, forced_cg_iterations=11, residual_reset_period=3)
    c = oracle_case(s, p)
    f = int(np.bincount(c["eg"]["frame"]).argmax())
    pert = dict(pose_offdiag=ltr.Perturb(drop_pose_offdiag=(f, (0, 4))), radius_x2=ltr.Perturb(radius_factor=2.0),
                stale_refresh=ltr.Perturb(stale_refresh=True))[which]
    radius = 1e-3 if which == "radius_x2" else p.initial_trust_region_radius
    assert _perturbed_ratio(c, p, pert, radius) > 1.0


def test_perturbation_breaks_candidate_bound(tiny_scene):
    """one E_r row missing moves the candidate cost by far more than the 1e-11 the GPU test allows"""
    s = tiny_scene
    p = _params(s)
    c = oracle_case(s, p)
    st = ltr.apply_step(c["state"], c["step"], c["R"].n, c["R"].F)
    ea = c["reg"][2]["raw_weight"]
    good = ltr.candidate_cost(s, st, c["eg"], c["reg"], ea, c["tw"])[0]
    bad = ltr.candidate_cost(s, st, c["eg"], c["reg"], ea, c["tw"], ltr.Perturb(drop_er_row=0))[0]
    assert abs(bad - good) > 1e-11 * abs(good)
