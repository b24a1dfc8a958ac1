"""Float64 restatement of one Levenberg-Marquardt trial of the engine: block-Jacobi preconditioner (k_cam_precond + the voxel
diagonal of k_cg_update), the PCG of k_cg_dir4 / k_cg_update / k_x_update and their scalar epilogues, the step delta = -s o x, the
model cost change, the candidate cost of k_candidate + k_eg_rows<ROWS_COST> + k_reg_cost, and the decision of k_lm_decide.

Its inputs are the quantities the kernels consumed: the rows of the iteration (normal_equations_ref.Rows), the gradient b, the
Jacobi scale s, jtj = s^2 colnorm^2 and the raw camera sums cam_acc.  Fed the engine's float32 values it measures the solve kernels'
arithmetic alone; fed the oracle's float64 values it reproduces the oracle's trial (tests/test_lm_trial_ref.py).

`pcg(..., f32=True)` is a float32 emulation of the same recurrence (float vectors, double dot products, the kernels' order of
operations, the operator product rounded once to float): its distance from the float64 result is the yardstick of the bound
    ||delta_gpu - delta_ref||_inf  <=  8 ||delta_emu - delta_ref||_inf + 2^-20 ||delta_ref||_inf       (per block)
that tests/test_gpu_lm_trial.py applies after two or more PCG iterations.
"""
from fractions import Fraction

import numpy as np
import scipy.sparse as sp

import normal_equations_ref as ner

U24 = ner.U24
# unknown blocks [sdf | albedo | poses | intr | dist]
BLOCKS = ("sdf", "albedo", "poses", "intr", "dist")


def blocks(n, F):
    """slices of the unknown vector per block"""
    o = (0, n, 2 * n, 2 * n + 6 * F, 2 * n + 6 * F + 4, 2 * n + 6 * F + 9)
    return {k: slice(o[i], o[i + 1]) for i, k in enumerate(BLOCKS)}


class Perturb:
    """Deliberate errors for the comparator's own test: one off-diagonal entry (a, b) of frame f's pose block dropped from the
    preconditioner, d^2 computed with the radius scaled by `radius_factor`, one E_r row missing from the candidate cost, and a
    residual refresh r = b - A x whose operator output still holds this iteration's A p (the qg the host clears before the refresh)."""

    def __init__(self, drop_pose_offdiag=None, radius_factor=None, drop_er_row=None, stale_refresh=False):
        self.drop_pose_offdiag, self.radius_factor = drop_pose_offdiag, radius_factor
        self.drop_er_row, self.stale_refresh = drop_er_row, stale_refresh


class System:
    """The trial's linear system  (S J^T W J S + D^2) x = b  and its block-Jacobi preconditioner.
    R: ner.Rows; s, b, jtj: [U]; cam_acc: [33F + 43] (ner.cam_sums layout); wg: the E_g type weight."""

    def __init__(self, R, s, b, jtj, cam_acc, wg):
        self.R, self.n, self.F, self.U = R, R.n, R.F, R.U
        J, _, _, w_op = R.matrix()
        self.s = np.asarray(s, np.float64)
        self.b = np.asarray(b, np.float64)
        self.jtj = np.asarray(jtj, np.float64)
        self.cam_acc = np.asarray(cam_acc, np.float64)
        self.wg = float(wg)
        self.K = (J.T @ sp.diags(w_op) @ J).tocsr()
        self.Kabs = (abs(J).T @ sp.diags(w_op) @ abs(J)).tocsr()

    def d2(self, P, radius, f32=False, perturb=None):
        """D^2 = clamp(jtj, min_lm_diagonal, max_lm_diagonal) / radius (float in k_cg_update / k_op_partial)"""
        if perturb is not None and perturb.radius_factor is not None:
            radius = radius * perturb.radius_factor
        if f32:
            dmin, dmax = np.float32(P.min_lm_diagonal), np.float32(min(P.max_lm_diagonal, 3.0e38))
            d = np.minimum(np.maximum(self.jtj.astype(np.float32), dmin), dmax)
            return (d * np.float32(1.0 / radius)).astype(np.float64)
        return np.minimum(np.maximum(self.jtj, P.min_lm_diagonal), P.max_lm_diagonal) / radius

    def precond(self, P, radius, perturb=None):
        """(voxel diagonal inverse [2n], camera block inverses [(base, m, inverse)], all blocks SPD).  Camera block of the unknowns
        base..base+m-1: w_g cam_acc_rc s_r s_c + d^2 on the diagonal (k_cam_precond), inverted in float64."""
        d2 = self.d2(P, radius, perturb=perturb)
        n, F = self.n, self.F
        vox = 1.0 / (self.jtj[:2 * n] + d2[:2 * n])
        cams, ok = [], True
        tail = 33 * F
        specs = [(2 * n + 6 * f, 6, 33 * f + 12) for f in range(F)] + [(2 * n + 6 * F, 4, tail + 18), (2 * n + 6 * F + 4, 5, tail + 28)]
        for bi, (base, m, t0) in enumerate(specs):
            A = np.zeros((m, m))
            k = t0
            for r in range(m):
                for c in range(r, m):
                    A[r, c] = A[c, r] = self.wg * self.cam_acc[k] * self.s[base + r] * self.s[base + c]
                    k += 1
            if perturb is not None and perturb.drop_pose_offdiag is not None and bi == perturb.drop_pose_offdiag[0]:
                a, c = perturb.drop_pose_offdiag[1]
                A[a, c] = A[c, a] = 0.0
            A[np.diag_indices(m)] += d2[base:base + m]
            try:
                np.linalg.cholesky(A)
                inv = np.linalg.inv(A)
            except np.linalg.LinAlgError:
                ok, inv = False, np.zeros((m, m))
            cams.append((base, m, inv))
        return vox, cams, ok


def pcg(S, P, radius, f32=False, perturb=None, apply_op=None, op_noise=None):
    """The PCG of one trial, from x = 0, r = b.  Returns dict(x, delta, it, status, zeta, zetas, Q1, xd2x, ok) where ok = False means
    a camera block of the preconditioner is not SPD (k_lm_decide: termination 3) and zetas[i - 1] is zeta after iteration i.
    f32: float32 emulation (see the module doc).  apply_op: v -> S J^T W J S v computed elsewhere (the engine's own operator kernels,
    Engine.debug_apply_operator), used in place of the float64 product.  op_noise = (c, seed): every product K (s o v) carries a
    random error uniform in +-c 2^-24 (|J|^T W |J| |s o v|)_j, the size test_gpu_normal_equations bounds the operator kernels' error by
    (c = rounding_counts(K)["q"]): a CPU stand-in for an operator summed in another order."""
    rd = (lambda v: np.asarray(v, np.float32).astype(np.float64)) if f32 else (lambda v: v)
    rs = (lambda v: float(np.float32(v))) if f32 else (lambda v: v)
    _, cams, ok = S.precond(P, radius, perturb)
    U, n2 = S.U, 2 * S.n
    d2 = S.d2(P, radius, f32, perturb)
    s, b = S.s, rd(S.b)
    vox_den = rd(S.jtj[:n2] + d2[:n2])          # z = r / (jtj + d^2) on the voxel unknowns
    rng = np.random.default_rng(op_noise[1]) if op_noise is not None else None

    def apply_m(r):
        z = np.empty(U)
        with np.errstate(divide="ignore", invalid="ignore"):
            z[:n2] = rd(r[:n2] / vox_den)
        for base, m, inv in cams:
            z[base:base + m] = rd(inv @ r[base:base + m])
        return z

    def op(v):
        """(q, v.q): q = s o float(K (s o v)) + d^2 o v"""
        if apply_op is not None:
            sq = np.asarray(apply_op(v), np.float64)
            return rd(sq + d2 * v), float(v @ sq + np.sum(d2 * v * v))
        vs = rd(s * v)
        kv = S.K @ vs
        if op_noise is not None:
            kv = kv + op_noise[0] * U24 * (S.Kabs @ np.abs(vs)) * rng.uniform(-1.0, 1.0, U)
        q = rd(s * rd(kv) + d2 * v)
        return q, float(vs @ kv + np.sum(d2 * v * v))

    out = dict(ok=ok, it=0, status=0, zeta=0.0, zetas=[], Q1=0.0, xd2x=0.0)
    x = np.zeros(U)
    r = b.copy()
    if not ok:
        out.update(x=x, delta=np.zeros(U))
        return out
    z = apply_m(r)
    rho = float(r @ z)
    forced = P.forced_cg_iterations
    max_it = forced if forced > 0 else P.max_linear_solver_iterations
    if rho == 0.0 or not np.isfinite(rho):
        out.update(x=x, delta=rd(-s * x), status=0 if rho == 0.0 else 1)
        return out
    p = np.zeros(U)
    beta = 0.0
    Q0, it = 0.0, 0
    while True:
        p = z.copy() if beta == 0.0 else rd(z + rs(beta) * p)
        q, pq = op(p)
        if pq <= 0.0 or np.isinf(pq):
            it += 1
            out["status"] = 2
            break
        alpha = rho / pq
        it += 1
        a = rs(alpha)
        x = rd(x + a * p)
        if it % P.residual_reset_period == 0:
            qx, _ = op(x)
            if perturb is not None and perturb.stale_refresh:
                qx = qx + (q - d2 * p)
            r = rd(b - qx)
        else:
            r = rd(r - a * q)
        z = apply_m(r)
        rho_new = float(r @ z)
        Q1 = -float(x @ (b + r))
        xd2x = float(np.sum(d2 * x * x))
        zeta = it * (Q1 - Q0) / Q1
        out.update(zeta=zeta, Q1=Q1, xd2x=xd2x)
        out["zetas"].append(zeta)
        stop = False
        if forced > 0:
            stop = it >= forced
        elif zeta < P.eta and it >= P.min_linear_solver_iterations:
            stop = True
        elif it >= max_it:
            stop, out["status"] = True, 3
        Q0 = Q1
        if stop:
            break
        beta = rho_new / rho
        rho = rho_new
        if rho_new == 0.0 or not np.isfinite(rho_new) or beta == 0.0 or not np.isfinite(beta):
            out["status"] = 1
            break
    out.update(x=x, delta=rd(-s * x), it=it)
    return out


def model_cost_change(R, delta):
    """-sum w m (f + m/2), m = J delta, over the rows of all four types (TrustRegionMinimizer's model cost change)"""
    J, res, w, _ = R.matrix()
    m = J @ np.asarray(delta, np.float64)
    return -float(np.sum(w * m * (res + 0.5 * m)))


def model_cost_change_bound(R, S, x, delta, K, d2):
    """Rounding part of the bound on |mcc_gpu - model_cost_change(R, delta)|, where the engine takes mcc = (x.D^2 x - Q1) / 2 =
    (x.D^2 x + x.(b + r)) / 2 from the PCG scalars (k_lm_decide).  Against the explicit value at its own delta it differs by
      (i)   the drift of the recursive residual r from b - A x: not bounded a priori, the caller adds 8 x the float32 emulation's
            |scalar - explicit| for it;
      (ii)  b's float error, |x|.(c_b 2^-24 M_b) with c_b = rounding_counts(K)["b"] and M_b the magnitude sums of b;
      (iii) the float operator weights (w_op = float(w), float type weights of the regulariser rows): 2 2^-24 sum w m^2;
      (iv)  d^2 in float (2 roundings): 2 2^-24 x.D^2 x;
      (v)   delta = float(-s o x) (1 rounding): 2^-24 sum_j |delta_j| (|J|^T W (|f| + |m|))_j.
    x, delta: float64 copies of the engine's x and delta; d2: the trial's D^2.  Returns the sum of (ii)-(v)."""
    J, res, w, _ = R.matrix()
    m = J @ delta
    Mb = S.s * (abs(J).T @ (w * np.abs(res)))
    cb = ner.rounding_counts(K)["b"]
    xd2x = float(np.sum(d2 * x * x))
    return U24 * (cb * float(np.abs(x) @ Mb) + 2 * float(np.sum(w * m * m)) + 2 * xd2x
                  + float(np.abs(delta) @ (abs(J).T @ (w * (np.abs(res) + np.abs(m))))))


def candidate_cost(scene, state, eg, reg, ea_w, type_w, perturb=None):
    """Cost of the frozen rows at `state` (dict sdf_refined, albedo, poses, intr, dist):
    E_g  sum raw_w r^2 over the rows (voxel, frame, raw_weight), r from oracle.eval_eg (invalid -> 0), the 10-voxel stencil
    E_r  sum lap^2 over the oracle's E_r voxels;  E_s  sum (sdf - sdf0)^2 over the E_s voxels, an exact 0 pinned to 1e-7
    E_a  sum w (a_v - a_b)^2 over the oracle's pairs with weights ea_w
    combined as 0.5 (w_g E_g + w_r E_r + w_s E_s + w_a E_a) like k_lm_decide.  Returns (cost, per-type raw sums)."""
    from oracle import eval_eg
    xyz = np.asarray(scene["xyz"], np.int64)
    idx = ner.VoxelIndex(xyz)
    sdf, alb = np.asarray(state["sdf_refined"], np.float64), np.asarray(state["albedo"], np.float64)
    poses, intr, dist = (np.asarray(state[k], np.float64) for k in ("poses", "intr", "dist"))
    vox = np.asarray(eg["voxel"], np.int64)
    frame = np.asarray(eg["frame"], np.int64)
    sdf_cols = np.stack([idx.lookup(vox, o) for o in ner.EG_SDF_OFFSETS], 1)
    alb_cols = np.stack([idx.lookup(vox, o) for o in ner.EG_ALB_OFFSETS], 1)
    lum = np.asarray(scene["lum"], np.float32)
    sh = np.asarray(scene["sh"], np.float64)
    vs, ps = float(np.float32(scene["voxel_size"])), float(scene.get("pyr_scale", 1.0))
    e_g = 0.0
    for i in range(len(vox)):
        r, _ = eval_eg(xyz[vox[i]], vs, ps, lum[frame[i]], sh[vox[i]], sdf[sdf_cols[i]], alb[alb_cols[i]], poses[frame[i]], intr, dist,
                       want_jac=False)
        e_g += float(eg["raw_weight"][i]) * r * r
    r1, r2, r3 = reg
    v = np.asarray(r1["voxel"], np.int64)
    if perturb is not None and perturb.drop_er_row is not None:
        v = np.delete(v, perturb.drop_er_row)
    nb = [sdf[idx.lookup(v, o)] for o in ner.FACE_OFFSETS]
    c = sdf[v]
    lap = ((nb[0] + nb[1] - 2.0 * c) + (nb[2] + nb[3] - 2.0 * c)) + (nb[4] + nb[5] - 2.0 * c)
    e_r = float(np.sum(lap * lap))
    v = np.asarray(r2["voxel"], np.int64)
    rs = sdf[v] - np.asarray(scene["sdf0"], np.float64)[v]
    rs = np.where(rs == 0.0, 1e-7, rs)
    e_s = float(np.sum(rs * rs))
    v, bb = np.asarray(r3["voxel"], np.int64), np.asarray(r3["aux"], np.int64)
    ra = alb[v] - alb[bb]
    e_a = float(np.sum(np.asarray(ea_w, np.float64) * ra * ra))
    sums = (e_g, e_r, e_s, e_a)
    return 0.5 * sum(t * x for t, x in zip(type_w, sums)), sums


def apply_step(state, delta, n, F):
    """state + float64(delta) per block (k_candidate)"""
    d = np.asarray(delta, np.float64)
    bl = blocks(n, F)
    return dict(sdf_refined=state["sdf_refined"] + d[bl["sdf"]], albedo=state["albedo"] + d[bl["albedo"]],
                poses=state["poses"] + d[bl["poses"]].reshape(F, 6), intr=state["intr"] + d[bl["intr"]], dist=state["dist"] + d[bl["dist"]])


def _one_minus_cube(t, fma):
    """1 - t^3 as k_lm_decide evaluates it (t2 = t*t, then one fused multiply-add), or with the cube rounded once (std::pow)"""
    if fma:
        return float(Fraction(1) - Fraction(t) * Fraction(t * t))
    return 1.0 - float(Fraction(t) ** 3)


def lm_decide(cost0, mcc, cand, step_norm, x_norm, radius, decrease_factor, lm_iterations, P, fma=True):
    """k_lm_decide for a valid step (finite, model_cost_change > 0), in plain double.  Returns dict(rho, radius, decrease_factor,
    termination, accepted, state) with state 'accepted', 'terminated' or 'running' (another trial follows)."""
    out = dict(rho=None, radius=radius, decrease_factor=decrease_factor, termination=2, accepted=False, state="running")
    if not (np.isfinite(step_norm) and mcc > 0.0):
        raise NotImplementedError("invalid steps are not restated")
    if step_norm <= P.parameter_tolerance * (x_norm + P.parameter_tolerance):
        out.update(termination=1, state="terminated")
        return out
    cost_change = cost0 - cand
    if abs(cost_change) <= P.function_tolerance * cost0:
        out.update(termination=1, state="terminated")
        return out
    rho = cost_change / mcc
    out["rho"] = rho
    if rho > P.min_relative_decrease:
        t = 2.0 * rho - 1.0
        r = min(P.max_trust_region_radius, radius / max(1.0 / 3.0, _one_minus_cube(t, fma)))
        out.update(radius=r, termination=0, accepted=True, state="accepted")
        return out
    r = radius / decrease_factor
    out.update(radius=r, decrease_factor=decrease_factor * 2.0)
    if r <= P.min_trust_region_radius:
        out.update(termination=1, state="terminated")
    elif lm_iterations >= P.lm_steps:
        out["state"] = "terminated"
    return out


def gradient_norms(R, free):
    """(max-norm, 2-norm) of the unscaled gradient J^T W f over the free unknowns"""
    J, res, w, _ = R.matrix()
    g = (J.T @ (w * res))[np.asarray(free, bool)]
    return float(np.abs(g).max()), float(np.sqrt(g @ g))


def block_compare(gpu, emus, ref, n, F, factor=8.0, floor=2.0 ** -20):
    """per block: ||gpu - ref||_inf / bound with bound = factor max_e ||emu_e - ref||_inf + floor ||ref||_inf over the float32
    emulations `emus` (one array or a list); a block whose ref is all zero must be exactly zero"""
    emus = [emus] if isinstance(emus, np.ndarray) else list(emus)
    out = {}
    for k, sl in blocks(n, F).items():
        g, r = (np.asarray(v, np.float64)[sl] for v in (gpu, ref))
        if not r.size:
            out[k] = 0.0
            continue
        err = float(np.abs(g - r).max())
        yard = max(float(np.abs(np.asarray(e, np.float64)[sl] - r).max()) for e in emus)
        bound = factor * yard + floor * float(np.abs(r).max())
        out[k] = (err / bound) if bound > 0 else (0.0 if err == 0 else np.inf)
    return out


def k1_bound(S, P, radius):
    """Componentwise bound of delta after ONE PCG iteration (x = alpha z, z = M^-1 b, p = z), |gpu - ref|_j <= c_j 2^-24 M_j with
    M_j = s_j |alpha| zmag_j, zmag_j = |z_j| on voxel unknowns and (|M^-1| |b|)_j on camera unknowns.  Float roundings on the chain:
      z (voxel)   d^2 = float(float(clamp(jtj)) * float(1/radius)) (2), + (1), / (1)                                      -> 4
      z (camera)  float(sum M^-1 r) in double (1) + the double Cholesky inverse, 2 m kappa 2^-53 relative              -> 1 + 2 m kappa 2^-29
      alpha       rho = r.z from float z: terms r_j z_j >= 0 (voxel) and r^T M^-1 r >= 0 per block, so rel <= the z count (4);
                  p.q = sum w u^2 + reg + sum d^2 p^2 with u = J (s o p) in float (c_u = 11: ps 1, four FMA chains of <= 8,
                  2 adds), wu = float(w u) (1), float weights (1), d^2 (2): rel <= (2 c_u sum w |u| U + 2 sum w u^2 + 3 sum d^2 p^2)
                  / p.q, U = |J| |s o p|; float(alpha) (1)
      x = float(alpha z) (1), delta = float(-s x) (1)
    Returns (ref delta, c_j 2^-24 M_j)."""
    _, cams, ok = S.precond(P, radius)
    assert ok
    n2 = 2 * S.n
    d2 = S.d2(P, radius)
    b, s = S.b, S.s
    z = np.empty(S.U)
    zmag = np.empty(S.U)
    cz = np.empty(S.U)
    z[:n2] = b[:n2] / (S.jtj[:n2] + d2[:n2])
    zmag[:n2] = np.abs(z[:n2])
    cz[:n2] = 4.0
    for base, m, inv in cams:
        sl = slice(base, base + m)
        z[sl] = inv @ b[sl]
        zmag[sl] = np.abs(inv) @ np.abs(b[sl])
        A = np.linalg.inv(inv)
        cz[sl] = 1.0 + 2 * m * np.linalg.cond(A) * 2.0 ** -29
    rho = float(b @ z)
    J, _, _, w_op = S.R.matrix()
    ps = s * z
    u = J @ ps
    Ub = abs(J) @ np.abs(ps)
    pq = float(np.sum(w_op * u * u) + np.sum(d2 * z * z))
    alpha = rho / pq
    pq_rel = float(2 * 11 * np.sum(w_op * np.abs(u) * Ub) + 2 * np.sum(w_op * u * u) + 3 * np.sum(d2 * z * z)) / pq
    c = cz + 4.0 + pq_rel + 1.0 + 2.0
    return -s * alpha * z, c * U24 * s * abs(alpha) * zmag
