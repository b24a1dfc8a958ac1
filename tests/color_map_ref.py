"""numpy statement of colour map optimisation of the keyframe poses (DESIGN.md §6y): measured on the CPU, not built on the device.

The samples are tests/distance_ref.py's face samples with tests/texture_ref.py's face normals; the observation weight is
tests/texture_ref.py's restatement of obs_probe / obs_finish (i3d_observe.cuh).  Every float operation is one numpy float32 operation
(IEEE round to nearest, no contraction) in a fixed order, as a kernel would use FA / FM / FD, so a device implementation can be held
byte-equal to the observation set, the intensities, the per-sample colours and the rows.  The per-keyframe systems are float64 sums
in numpy's order, and the solve is track_ref's Cholesky and Rodrigues update in Python floats.

Row functions take the float type `ft`: float32 is the statement, float64 evaluates the same formulas for the finite-difference
checks of the Jacobian.
"""
from __future__ import annotations

import math

import numpy as np

import distance_ref
import texture_ref
import track_ref

f32 = np.float32
VALS = 29
UPPER = track_ref.UPPER
# per-keyframe status of a solve
OK, FIXED, FEW_ROWS, NOT_PD, NON_FINITE = 0, 1, 2, 3, 4
# the loop's parameters; samples_per_edge (L) and max_occlusion_distance (1 and 0.02 by default) belong to Problem
DEFAULTS = dict(iterations=30, min_views=2, min_rows=64, lam=1e-4, stop_rotation=1e-6, stop_translation=1e-7)


def params(**over):
    p = dict(DEFAULTS)
    p.update(over)
    return p


def pose_rt64(poses):
    """The engine camera's poses as world -> camera R | t [F, 12] in double: k_pose_mats' rule (math::poseVecAAToMat) without the cast."""
    poses = np.asarray(poses, np.float64)
    out = np.zeros((len(poses), 12))
    for f, p in enumerate(poses):
        wx, wy, wz = (float(a) for a in p[:3])
        n2 = wx * wx + wy * wy + wz * wz
        angle = math.sqrt(n2)
        ax, ay, az = (wx / angle, wy / angle, wz / angle) if n2 > 0.0 else (wx, wy, wz)
        s, c = math.sin(angle), math.cos(angle)
        sx, sy, sz = s * ax, s * ay, s * az
        c1x, c1y, c1z = (1.0 - c) * ax, (1.0 - c) * ay, (1.0 - c) * az
        M = [0.0] * 9
        t = c1x * ay; M[1] = t - sz; M[3] = t + sz
        t = c1x * az; M[2] = t + sy; M[6] = t - sy
        t = c1y * az; M[5] = t - sx; M[7] = t + sx
        M[0] = c1x * ax + c; M[4] = c1y * ay + c; M[8] = c1z * az + c
        out[f, :9] = M
        out[f, 9:] = p[3:]
    return out


def samples(mesh, L):
    """points float32 [S, 3] (distance_ref's rule and order), normals float32 [S, 3] (the bake's face normal) and valid [S] (non-zero
    normal)"""
    P, _ = distance_ref.samples(mesh, L)
    V = np.asarray(mesh["vertices"], f32).reshape(-1, 3)
    Fc = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    N = np.repeat(texture_ref.face_normals(V, Fc), L * L, axis=0)
    return P, N, ~np.all(N == 0, 1)


def project(q, cam, ft=f32):
    """(x, y) normalised, (pu, pv) pixel of camera points q (list of 3 arrays of type ft): obs_probe's projection with distortion"""
    c = lambda a: ft(a)
    d = [c(a) for a in cam["d"]]
    with np.errstate(all="ignore"):
        x, y = q[0] / q[2], q[1] / q[2]
        xd, yd = x, y
        if any(a != 0 for a in d):
            r2 = x * x + y * y
            r4 = r2 * r2
            r6 = r4 * r2
            dc = ((c(1) + d[0] * r2) + d[1] * r4) + d[2] * r6
            xd = (x * dc + ((c(2) * d[3]) * x) * y) + d[4] * (r2 + (c(2) * x) * x)
            yd = (y * dc + ((c(2) * d[4]) * xd) * y) + d[3] * (r2 + (c(2) * y) * y)
        return x, y, xd, yd, c(cam["fx"]) * xd + c(cam["cx"]), c(cam["fy"]) * yd + c(cam["cy"])


def proj_jacobian(q, cam, ft=f32):
    """the distortion Jacobian (dxx, dxy, dyx, dyy) of (xd, yd) over the normalised (x, y), and x, y; row() folds it with the
    intrinsics and the image gradient"""
    c = lambda a: ft(a)
    d = [c(a) for a in cam["d"]]
    x, y, xd, yd, _, _ = project(q, cam, ft)
    if not any(a != 0 for a in d):
        one, zero = np.ones_like(x), np.zeros_like(x)
        return one, zero, zero, one, x, y
    with np.errstate(all="ignore"):
        r2 = x * x + y * y
        r4 = r2 * r2
        r6 = r4 * r2
        dc = ((c(1) + d[0] * r2) + d[1] * r4) + d[2] * r6
        dcr = (d[0] + (c(2) * d[1]) * r2) + (c(3) * d[2]) * r4
        dxx = ((dc + ((c(2) * x) * x) * dcr) + (c(2) * d[3]) * y) + (c(6) * d[4]) * x
        dxy = ((((c(2) * x) * y) * dcr) + (c(2) * d[3]) * x) + (c(2) * d[4]) * y
        dyx = ((((c(2) * x) * y) * dcr) + ((c(2) * d[4]) * y) * dxx) + (c(2) * d[3]) * x
        dyy = ((dc + ((c(2) * y) * y) * dcr) + (c(2) * d[4]) * (xd + y * dxy)) + (c(6) * d[3]) * y
    return dxx, dxy, dyx, dyy, x, y


def sample_image(lum, pu, pv, ft=f32, grad=True):
    """(inside, I, gu, gv): the bilinear value at (pu, pv) (pixel centres at integers) and the same blend of the central differences at
    the four corner pixels; inside = all 4 x 4 taps in the image"""
    c = lambda a: ft(a)
    H, W = lum.shape
    img = lum.astype(ft)
    with np.errstate(all="ignore"):
        fx0, fy0 = np.floor(pu), np.floor(pv)
        inside = np.isfinite(fx0) & np.isfinite(fy0)
        x0 = np.where(inside, fx0, 0).astype(np.int64)
        y0 = np.where(inside, fy0, 0).astype(np.int64)
    inside &= (x0 >= 1) & (x0 + 2 <= W - 1) & (y0 >= 1) & (y0 + 2 <= H - 1)
    x0, y0 = np.where(inside, x0, 1), np.where(inside, y0, 1)
    ax, ay = (pu - fx0).astype(ft), (pv - fy0).astype(ft)
    ax, ay = np.where(inside, ax, c(0)), np.where(inside, ay, c(0))
    bx, by = c(1) - ax, c(1) - ay
    w = ((bx * by, 0, 0), (ax * by, 1, 0), (bx * ay, 0, 1), (ax * ay, 1, 1))
    tap = lambda dx, dy: img[y0 + dy, x0 + dx]
    I = np.zeros_like(ax)
    for wk, dx, dy in w:
        I = I + wk * tap(dx, dy)
    if not grad:
        return inside, I, None, None
    gu, gv = np.zeros_like(ax), np.zeros_like(ax)
    half = c(0.5)
    for wk, dx, dy in w:
        gu = gu + wk * (half * (tap(dx + 1, dy) - tap(dx - 1, dy)))
    for wk, dx, dy in w:
        gv = gv + wk * (half * (tap(dx, dy + 1) - tap(dx, dy - 1)))
    return inside, I, gu, gv


def observe(P, N, valid, T, cam, lum, depth, occlusion, grad=False):
    """Per sample at the world -> camera pose T (double [12]): weight w (0 = not observed), I, gu, gv, q (list of 3) of keyframe
    (lum, depth)"""
    rt = np.asarray(T, np.float64).astype(f32)
    q, pu, pv, d, ok = texture_ref.probe(P, rt, cam, depth)
    w = texture_ref.weight(q, d, ok, N, rt, occlusion)
    w = np.where(valid, w, f32(0))
    inside, I, gu, gv = sample_image(lum, pu, pv, f32, grad)
    w = np.where(inside, w, f32(0)).astype(f32)
    return w, I, gu, gv, [q[:, 0], q[:, 1], q[:, 2]]


def row(q, gu, gv, cam, ft=f32):
    """J [m, 6] (d r / d(w, v) of T <- [Rodrigues(w) | v] T at 0) from camera points q and image gradients"""
    c = lambda a: ft(a)
    dxx, dxy, dyx, dyy, x, y = proj_jacobian(q, cam, ft)
    with np.errstate(all="ignore"):
        a = gu * c(cam["fx"])
        b = gv * c(cam["fy"])
        gx = a * dxx + b * dyx
        gy = a * dxy + b * dyy
        iz = c(1) / q[2]
        g0, g1 = gx * iz, gy * iz
        g2 = -((gx * x + gy * y) * iz)
        J = [q[1] * g2 - q[2] * g1, q[2] * g0 - q[0] * g2, q[0] * g1 - q[1] * g0, g0, g1, g2]
    return np.stack(J, 1).astype(ft)


def residual(P, T, cam, lum, C, ft=np.float64):
    """r = I(pi(T P)) - C in type ft, for the finite-difference checks (no weight, no gates)"""
    T = np.asarray(T, np.float64)
    q = [((ft(T[3 * k]) * P[:, 0].astype(ft) + ft(T[3 * k + 1]) * P[:, 1].astype(ft)) + ft(T[3 * k + 2]) * P[:, 2].astype(ft)) + ft(T[9 + k])
         for k in range(3)]
    _, _, _, _, pu, pv = project(q, cam, ft)
    _, I, _, _ = sample_image(lum, pu, pv, ft, grad=False)
    return I - C


class Problem:
    """The samples of one mesh and the keyframes (lum, depth [F, H, W], float camera dict of render_ref.camera)"""

    def __init__(self, mesh, lum, depth, cam, L=1, occlusion=0.02):
        self.P, self.N, self.valid = samples(mesh, L)
        self.lum, self.depth = np.asarray(lum, f32), np.asarray(depth, f32)
        self.cam, self.occ = cam, f32(occlusion)
        self.F = len(self.lum)

    def colours(self, T, min_views):
        """(C float32 [S] with NaN for unused samples, views [S], W [S, F], I [S, F])"""
        S, F = len(self.P), self.F
        W, I = np.zeros((S, F), f32), np.zeros((S, F), f32)
        for k in range(F):
            W[:, k], I[:, k], _, _, _ = observe(self.P, self.N, self.valid, T[k], self.cam, self.lum[k], self.depth[k], self.occ)
        obs = W > 0
        num, den = np.zeros(S), np.zeros(S)
        for k in range(F):
            num = num + np.where(obs[:, k], W[:, k].astype(np.float64) * I[:, k].astype(np.float64), 0.0)
            den = den + np.where(obs[:, k], W[:, k].astype(np.float64), 0.0)
        views = obs.sum(1)
        with np.errstate(all="ignore"):
            C = np.where(views >= min_views, (num / den).astype(f32), f32(np.nan)).astype(f32)
        return C, views, W, I

    def rows(self, T, k, C):
        """(w, r, J) float32 of keyframe k's rows (one per used sample it observes)"""
        w, I, gu, gv, q = observe(self.P, self.N, self.valid, T[k], self.cam, self.lum[k], self.depth[k], self.occ, grad=True)
        m = (w > 0) & ~np.isnan(C)
        J = row([a[m] for a in q], gu[m], gv[m], self.cam)
        return w[m], (I[m] - C[m]).astype(f32), J

    def system(self, T, k, C):
        """the 29 doubles of keyframe k: upper J^T W J, J^T W r, sum w r^2, rows"""
        w, r, J = self.rows(T, k, C)
        wd, rd, Jd = w.astype(np.float64), r.astype(np.float64), J.astype(np.float64)
        S = np.zeros(VALS)
        for j, (a, b) in enumerate(UPPER):
            S[j] = ((wd * Jd[:, a]) * Jd[:, b]).sum()
        for a in range(6):
            S[21 + a] = ((wd * Jd[:, a]) * rd).sum()
        S[27] = ((wd * rd) * rd).sum()
        S[28] = len(w)
        return S


def solve(S, lam):
    """(status, xi) of (A + lam diag(A)) xi = -b"""
    S = [float(a) for a in S]
    if not all(math.isfinite(a) for a in S):
        return NON_FINITE, None
    D = list(S)
    j = 0
    for a in range(6):
        for b in range(a, 6):
            if a == b:
                D[j] = S[j] + lam * S[j]
            j += 1
    st, x = track_ref.solve(D)
    if st:
        return (NOT_PD if st == 2 else NON_FINITE), None
    return OK, x


def step(prob, T, fixed, p):
    """One iteration: colours, systems, solves.  Returns (T_new, status [F], systems [F, 29], C, xi norms (|w|, |v|) [F, 2])"""
    C, _, _, _ = prob.colours(T, p["min_views"])
    F = prob.F
    Tn = [list(map(float, t)) for t in T]
    status = np.zeros(F, np.int32)
    sys = np.zeros((F, VALS))
    norms = np.zeros((F, 2))
    for k in range(F):
        sys[k] = prob.system(T, k, C)
        if fixed[k]:
            status[k] = FIXED
            continue
        if sys[k, 28] < p["min_rows"]:
            status[k] = FEW_ROWS
            continue
        st, x = solve(sys[k], p["lam"])
        if st:
            status[k] = st
            continue
        Tk = track_ref.update(Tn[k], x)
        if not all(math.isfinite(a) for a in list(x) + Tk):
            status[k] = NON_FINITE
            continue
        Tn[k] = Tk
        norms[k] = math.sqrt((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]), math.sqrt((x[3] * x[3] + x[4] * x[4]) + x[5] * x[5])
    return np.array(Tn), status, sys, C, norms


def optimize(prob, T0, fixed=None, **over):
    """The whole call: returns (T [F, 12], status [F], info dict, C at the final poses, systems at the final poses)"""
    p = params(**over)
    F = prob.F
    fixed = np.zeros(F, bool) if fixed is None else np.asarray(fixed, bool)
    T = np.array(T0, np.float64)
    status = np.where(fixed, FIXED, OK).astype(np.int32)
    energy_before, it = None, 0
    for it in range(1, p["iterations"] + 1):
        T, status, sys, _, norms = step(prob, T, fixed, p)
        if energy_before is None:
            energy_before = sys[:, 27].sum()
        moved = status == OK
        if np.all((norms[moved, 0] < p["stop_rotation"]) & (norms[moved, 1] < p["stop_translation"])):
            break
    else:
        it = p["iterations"]
    C, views, _, _ = prob.colours(T, p["min_views"])
    sys = np.stack([prob.system(T, k, C) for k in range(F)])
    if energy_before is None:
        energy_before = sys[:, 27].sum()
    info = dict(iterations=it, energy_before=float(energy_before), energy_after=float(sys[:, 27].sum()), rows=int(sys[:, 28].sum()),
                samples=len(prob.P), samples_used=int((~np.isnan(C)).sum()))
    return T, status, info, C, sys
