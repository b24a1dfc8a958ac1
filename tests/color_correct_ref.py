"""numpy statement of the per-keyframe colour gain estimate and its correction (DESIGN.md §6z).

Shares no code with the kernels.  Every float32 operation is one numpy float32 operation and every float64 operation one numpy float64
operation (IEEE round to nearest, no contraction), in the order stated here, so the device can be held byte-equal to the observations, the
fixed-point bin sums and the corrected frames, and to the fields to the last bit of the fixed-order solve.

Model: keyframe k's channel ch (B, G, R) of the colour frame at pixel u is exp(l_k,ch(u) + x_s,ch) for the surface sample s it sees,
with l a uniform cubic B-spline over control points `spacing` px apart and x a per-sample log colour.

* samples: tests/color_map_ref.py's (distance_ref's sub-triangle centroids, the bake's face normal, a zero normal drops the sample).
* observations: texture_ref.probe / weight (obs_probe / obs_finish) at the float pose; c = the float32 bilinear value of each uint8
  channel at (pu, pv), pixel centres at integers, all four taps in the image: ((bx by) c00 + (ax by) c10) + (bx ay) c01) + (ax ay) c11.
  An observation counts when w > 0 and all three c lie in [c_min, 254]; its bin is (iu // b, iv // b) of probe's rounded pixel.
* log: LOG(c) below, a fixed sequence of float64 operations (frexp, then an atanh series), so the device computes the same bits.
* spline: control grid Gy x Gx = (H // spacing + 4) x (W // spacing + 4).  A pixel range [lo, hi) maps to x = (lo + hi) / (2 spacing);
  a bin is its clipped pixel range, a pixel u is [u, u + 1).  Cell i = floor(x), t = x - i, l = sum_a By_a (sum_b Bx_b C[j + a, i + b]).
* sweep: (1) x_s = sum_k w (L - l_k(bin)) / sum_k w over the samples seen by >= min_views keyframes, in frame order; (2) per keyframe the
  bin sums Qw = sum rint(w 2^32) and Qwt = sum rint(w t 2^28) of t = clamp(L - x_s, -8, 8) (integers: order free), then
  A = sum_bins (W beta_p) beta_q (bins in row-major order) + lam_s D^T D + lam_0 I, b_ch = sum_bins T_ch beta, solved by Cholesky
  (left-looking, sums in index order).  A keyframe with fewer than min_obs observations keeps l = 0 (FEW_OBS); a failed Cholesky keeps
  its previous field (NOT_PD).
* gauge: after the last sweep, subtract from the OK keyframes' control values each channel's mean over them (summed in (k, j, i) order).
* apply: c' = rint(min(max(c EXP(-l(pixel)), 0), 255)), EXP below.
"""
from __future__ import annotations

import math

import numpy as np

import color_map_ref as cm
import texture_ref

f32, f64 = np.float32, np.float64
OK, FEW_OBS, NOT_PD = 0, 1, 2
W_SCALE = 2.0 ** 32            # Qw = rint(w 2^32) <= 2^32 per observation (w <= 1)
WT_SCALE = 2.0 ** 28           # Qwt = rint(w t 2^28), |t| <= 8 so |Qwt| <= 2^31: a bin overflows int64 only past 2^31 observations
T_CLAMP = 8.0
LN2 = 0.6931471805599453
DEFAULTS = dict(L=1, occlusion=0.02, spacing=64, bin=8, sweeps=4, min_views=2, min_obs=256, lam_s=0.01, lam_0=1e-4, c_min=8.0,
                flat=0.0, flat_r=2)


def params(**over):
    p = dict(DEFAULTS)
    p.update(over)
    return p


# ---------------------------------------------------------------------------------------------------------------------- log and exp
_LOG_C = [1.0 / (2 * n + 1) for n in range(10, -1, -1)]         # 1/21, 1/19, ..., 1/3, 1
_EXP_N = list(range(16, 0, -1))


def LOG(c):
    """log of positive float64 c: c = m 2^e with m in [sqrt(1/2), sqrt(2)), s = (m - 1) / (m + 1), log m = 2 s P(s^2)."""
    c = np.asarray(c, f64)
    m, e = np.frexp(c)                                           # m in [0.5, 1)
    lo = m < 0.7071067811865476
    m = np.where(lo, m * 2.0, m)
    e = np.where(lo, e - 1, e).astype(f64)
    s = (m - 1.0) / (m + 1.0)
    z = s * s
    p = np.full_like(s, _LOG_C[0])
    for k in _LOG_C[1:]:
        p = p * z + k
    return e * LN2 + (2.0 * s) * p


def EXP(x):
    """exp of float64 x: k = rint(x / ln 2), r = x - k ln 2, Horner of the Taylor series to r^16 / 16!, times 2^k."""
    x = np.asarray(x, f64)
    k = np.rint(x / LN2)
    r = x - k * LN2
    p = np.ones_like(r)
    for n in _EXP_N:
        p = 1.0 + (r * p) / float(n)
    return np.ldexp(p, k.astype(np.int64))


# ---------------------------------------------------------------------------------------------------------------------- B-spline
def grid_shape(W, H, spacing):
    return H // spacing + 4, W // spacing + 4


def basis(lo, hi, spacing):
    """(cell, [B0, B1, B2, B3]) float64 of pixel ranges [lo, hi) (integer arrays)."""
    x = (np.asarray(lo, f64) + np.asarray(hi, f64)) / (2.0 * spacing)
    i = np.floor(x)
    t = x - i
    t2 = t * t
    t3 = t2 * t
    u = 1.0 - t
    B = [((u * u) * u) / 6.0, ((3.0 * t3 - 6.0 * t2) + 4.0) / 6.0, (((-3.0 * t3 + 3.0 * t2) + 3.0 * t) + 1.0) / 6.0, t3 / 6.0]
    return i.astype(np.int64), B


def evaluate(C, ix, Bx, iy, By):
    """l at points with column basis (ix, Bx) and row basis (iy, By): sum_a By_a (sum_b Bx_b C[iy + a, ix + b]), broadcast."""
    out = None
    for a in range(4):
        row = None
        for b in range(4):
            v = Bx[b] * C[iy + a, ix + b]
            row = v if row is None else row + v
        v = By[a] * row
        out = v if out is None else out + v
    return out


def bin_basis(W, H, spacing, b):
    """Per bin column / row: (cell, basis) of its clipped pixel range."""
    def axis(n):
        lo = np.arange(0, n, b)
        return basis(lo, np.minimum(lo + b, n), spacing)
    return axis(W), axis(H)


def field_at_bins(C, W, H, spacing, b):
    """l [By, Bx] of control grid C at every bin."""
    (ix, Bx), (iy, By) = bin_basis(W, H, spacing, b)
    return evaluate(C, ix[None, :], [v[None, :] for v in Bx], iy[:, None], [v[:, None] for v in By])


def field_at_pixels(C, W, H, spacing):
    ix, Bx = basis(np.arange(W), np.arange(W) + 1, spacing)
    iy, By = basis(np.arange(H), np.arange(H) + 1, spacing)
    return evaluate(C, ix[None, :], [v[None, :] for v in Bx], iy[:, None], [v[:, None] for v in By])


def second_differences(Gy, Gx):
    """D^T D (float64, integer entries) of the second differences along rows and columns of a Gy x Gx grid, index j Gx + i."""
    n = Gy * Gx
    rows = []
    for j in range(Gy):
        for i in range(1, Gx - 1):
            rows.append(((j * Gx + i - 1, 1.0), (j * Gx + i, -2.0), (j * Gx + i + 1, 1.0)))
    for j in range(1, Gy - 1):
        for i in range(Gx):
            rows.append((((j - 1) * Gx + i, 1.0), (j * Gx + i, -2.0), ((j + 1) * Gx + i, 1.0)))
    R = np.zeros((n, n))
    for r in rows:
        for p, a in r:
            for q, c in r:
                R[p, q] += a * c
    return R


# ---------------------------------------------------------------------------------------------------------------------- observations
def bilinear(img, pu, pv):
    """(inside, c float32 [m, 3]) of the uint8 B, G, R image at (pu, pv)."""
    H, W = img.shape[:2]
    with np.errstate(all="ignore"):
        fx0, fy0 = np.floor(pu), np.floor(pv)
        inside = np.isfinite(fx0) & np.isfinite(fy0)
        inside &= (fx0 >= 0) & (fx0 <= W - 2) & (fy0 >= 0) & (fy0 <= H - 2)
        x0 = np.where(inside, fx0, 0).astype(np.int64)
        y0 = np.where(inside, fy0, 0).astype(np.int64)
        ax = np.where(inside, pu - fx0, f32(0)).astype(f32)
        ay = np.where(inside, pv - fy0, f32(0)).astype(f32)
    bx, by = f32(1) - ax, f32(1) - ay
    w00, w10, w01, w11 = bx * by, ax * by, bx * ay, ax * ay
    t = lambda dx, dy: img[y0 + dy, x0 + dx].astype(f32)
    c = ((w00[:, None] * t(0, 0) + w10[:, None] * t(1, 0)) + w01[:, None] * t(0, 1)) + w11[:, None] * t(1, 1)
    return inside, c.astype(f32)


def flat(img, pu, pv, ratio, r):
    """The measured variant's gate (off by default): every channel's max <= ratio * min over the pixels x0 - r .. x0 + 1 + r,
    y0 - r .. y0 + 1 + r around the bilinear footprint (clamped to the image).  It drops observations near albedo edges, where a
    sub-pixel misregistration of the mesh changes the colour far more than the gain does."""
    H, W = img.shape[:2]
    with np.errstate(all="ignore"):
        x0 = np.clip(np.nan_to_num(np.floor(pu)), 0, W - 2).astype(np.int64)
        y0 = np.clip(np.nan_to_num(np.floor(pv)), 0, H - 2).astype(np.int64)
    lo, hi = np.full((len(pu), 3), 255.0), np.zeros((len(pu), 3))
    for dy in range(-r, 2 + r):
        for dx in range(-r, 2 + r):
            v = img[np.clip(y0 + dy, 0, H - 1), np.clip(x0 + dx, 0, W - 1)].astype(f64)
            lo, hi = np.minimum(lo, v), np.maximum(hi, v)
    return np.all(hi <= ratio * lo, 1)


class Problem:
    """The samples of one mesh, the keyframes' depth [F, H, W] and colour [F, H, W, 3] (B, G, R), float poses [F, 12] and the camera."""

    def __init__(self, mesh, depth, bgr, rt, cam, **over):
        self.p = params(**over)
        p = self.p
        self.P, self.N, self.valid = cm.samples(mesh, p["L"])
        depth, bgr = np.asarray(depth, f32), np.asarray(bgr, np.uint8)
        rt = np.asarray(rt, f32)
        self.bgr = bgr
        self.F, self.H, self.W = depth.shape
        S, F, b = len(self.P), self.F, p["bin"]
        self.Bx, self.By = -(-self.W // b), -(-self.H // b)
        self.w = np.zeros((S, F), f32)
        self.bin = np.zeros((S, F), np.int64)
        self.L = np.zeros((S, F, 3))
        cmin = f32(p["c_min"])
        for k in range(F):
            q, pu, pv, d, ok = texture_ref.probe(self.P, rt[k], cam, depth[k])
            w = texture_ref.weight(q, d, ok, self.N, rt[k], p["occlusion"])
            w = np.where(self.valid, w, f32(0))
            inside, c = bilinear(bgr[k], pu, pv)
            good = inside & (w > 0) & np.all((c >= cmin) & (c <= f32(254)), 1)
            if p["flat"] > 0:
                good &= flat(bgr[k], pu, pv, p["flat"], p["flat_r"])
            self.w[:, k] = np.where(good, w, f32(0))
            with np.errstate(all="ignore"):
                iu = np.where(good, np.trunc(pu + f32(0.5)), 0).astype(np.int64)
                iv = np.where(good, np.trunc(pv + f32(0.5)), 0).astype(np.int64)
            self.bin[:, k] = (iv // b) * self.Bx + iu // b
            self.L[:, k] = np.where(good[:, None], LOG(np.where(good[:, None], c, f32(1)).astype(f64)), 0.0)
        self.obs = self.w > 0
        self.views = self.obs.sum(1)
        self.used = self.views >= p["min_views"]
        self.Gy, self.Gx = grid_shape(self.W, self.H, p["spacing"])
        (self.bix, self.bBx), (self.biy, self.bBy) = bin_basis(self.W, self.H, p["spacing"], b)
        self.R = second_differences(self.Gy, self.Gx)

    # the three blocks -------------------------------------------------------------------------------------------------------------
    def bin_fields(self, C):
        """l_k,ch at every bin, float64 [F, 3, By * Bx]"""
        return np.stack([[field_at_bins(C[k, ch], self.W, self.H, self.p["spacing"], self.p["bin"]).ravel() for ch in range(3)]
                         for k in range(self.F)])

    def colours(self, C):
        """x float64 [S, 3] (NaN for unused samples) in frame order"""
        lb = self.bin_fields(C)
        S = len(self.P)
        num, den = np.zeros((S, 3)), np.zeros(S)
        for k in range(self.F):
            o = self.obs[:, k]
            wd = self.w[:, k].astype(f64)
            l = lb[k][:, self.bin[:, k]].T
            num = np.where(o[:, None], num + wd[:, None] * (self.L[:, k] - l), num)
            den = np.where(o, den + wd, den)
        with np.errstate(all="ignore"):
            x = num / den[:, None]
        return np.where(self.used[:, None], x, np.nan)

    def bin_sums(self, x):
        """(Qw uint64 [F, nbins], Qwt int64 [F, 3, nbins], observations [F]) of the used samples' observations"""
        nb = self.Bx * self.By
        Qw = np.zeros((self.F, nb), np.uint64)
        Qwt = np.zeros((self.F, 3, nb), np.int64)
        nobs = np.zeros(self.F, np.int64)
        for k in range(self.F):
            o = self.obs[:, k] & self.used
            wd = self.w[o, k].astype(f64)
            t = np.clip(self.L[o, k] - x[o], -T_CLAMP, T_CLAMP)
            qw = np.rint(wd * W_SCALE).astype(np.uint64)
            qwt = np.rint((wd[:, None] * t) * WT_SCALE).astype(np.int64)
            np.add.at(Qw[k], self.bin[o, k], qw)
            for ch in range(3):
                np.add.at(Qwt[k, ch], self.bin[o, k], qwt[:, ch])
            nobs[k] = o.sum()
        return Qw, Qwt, nobs

    def system(self, Qw, Qwt):
        """(A [n, n], b [3, n]) float64 of one keyframe's bin sums"""
        Gx, n = self.Gx, self.Gy * self.Gx
        A, rhs = np.zeros((n, n)), np.zeros((3, n))
        Wb = Qw.astype(f64) / W_SCALE
        Tb = Qwt.astype(f64) / WT_SCALE
        for bi in np.nonzero(Qw)[0]:
            by, bx = divmod(int(bi), self.Bx)
            i, j = int(self.bix[bx]), int(self.biy[by])
            beta = np.array([self.bBy[a][by] * self.bBx[c][bx] for a in range(4) for c in range(4)])
            idx = np.array([(j + a) * Gx + i + c for a in range(4) for c in range(4)])
            A[np.ix_(idx, idx)] = A[np.ix_(idx, idx)] + (Wb[bi] * beta)[:, None] * beta[None, :]
            rhs[:, idx] = rhs[:, idx] + Tb[:, bi][:, None] * beta[None, :]
        A = A + self.p["lam_s"] * self.R
        A[np.arange(n), np.arange(n)] += self.p["lam_0"]
        return A, rhs

    def sweep(self, C):
        """One sweep from control grids C [F, 3, Gy, Gx]: (C', status [F], x, nobs [F], Qw, Qwt)"""
        x = self.colours(C)
        Qw, Qwt, nobs = self.bin_sums(x)
        Cn = C.copy()
        status = np.zeros(self.F, np.int32)
        for k in range(self.F):
            if nobs[k] < self.p["min_obs"]:
                Cn[k] = 0.0
                status[k] = FEW_OBS
                continue
            A, rhs = self.system(Qw[k], Qwt[k])
            sol = cholesky_solve(A, rhs)
            if sol is None:
                status[k] = NOT_PD
                continue
            Cn[k] = sol.reshape(3, self.Gy, self.Gx)
        return Cn, status, x, nobs, Qw, Qwt

    def energy(self, C, x):
        """sum w (L - l - x)^2 over the used samples' observations + the regularisers, float64 (for the tests)"""
        lb = self.bin_fields(C)
        e = 0.0
        for k in range(self.F):
            o = self.obs[:, k] & self.used
            r = self.L[o, k] - lb[k][:, self.bin[o, k]].T - x[o]
            e += float((self.w[o, k].astype(f64)[:, None] * r * r).sum())
        n = self.Gy * self.Gx
        for k in range(self.F):
            for ch in range(3):
                c = C[k, ch].ravel()
                e += self.p["lam_s"] * float(c @ self.R @ c) + self.p["lam_0"] * float(c @ c)
        return e


def cholesky_solve(A, rhs):
    """Left-looking Cholesky A = L L^T (column j: acc = A[j:, j] - sum_k<j L[j:, k] L[j, k] in k order, L[j, j] = sqrt(acc[0]),
    L[j:, j] = acc / L[j, j]), then L y = b and L^T z = y with sums in index order.  None when a pivot is not positive."""
    n = len(A)
    Lm = np.zeros((n, n))
    for j in range(n):
        acc = A[j:, j].copy()
        for k in range(j):
            acc = acc - Lm[j:, k] * Lm[j, k]
        if not acc[0] > 0.0:
            return None
        d = math.sqrt(acc[0])
        Lm[j:, j] = acc / d
    y = np.zeros_like(rhs)
    for i in range(n):
        acc = rhs[:, i].copy()
        for k in range(i):
            acc = acc - Lm[i, k] * y[:, k]
        y[:, i] = acc / Lm[i, i]
    z = np.zeros_like(rhs)
    for i in range(n - 1, -1, -1):
        acc = y[:, i].copy()
        for k in range(i + 1, n):
            acc = acc - Lm[k, i] * z[:, k]
        z[:, i] = acc / Lm[i, i]
    return z


def gauge(C, status):
    """Subtract each channel's mean over the OK keyframes' control values, summed in (k, j, i) order."""
    C = C.copy()
    ok = status == OK
    if not ok.any():
        return C
    for ch in range(3):
        s = 0.0
        for k in np.nonzero(ok)[0]:
            for v in C[k, ch].ravel():
                s = s + float(v)
        m = s / float(ok.sum() * C.shape[2] * C.shape[3])
        C[ok, ch] = C[ok, ch] - m
    return C


def estimate(prob, trace=False):
    """The whole estimate: (C [F, 3, Gy, Gx] float64, status [F], nobs [F], info dict[, per-sweep energies])"""
    C = np.zeros((prob.F, 3, prob.Gy, prob.Gx))
    energies = []
    status = nobs = None
    for _ in range(prob.p["sweeps"]):
        if trace:
            energies.append(prob.energy(C, prob.colours(C)))
        C, status, x, nobs, _, _ = prob.sweep(C)
        if trace:
            energies.append(prob.energy(C, x))
    C = gauge(C, status)
    info = dict(samples=len(prob.P), samples_used=int(prob.used.sum()), observations=int(nobs.sum()), grid_x=prob.Gx, grid_y=prob.Gy)
    return (C, status, nobs, info, energies) if trace else (C, status, nobs, info)


def apply(bgr, C, spacing):
    """Corrected frames: c' = rint(min(max(c EXP(-l), 0), 255)) per pixel and channel."""
    bgr = np.asarray(bgr, np.uint8)
    F, H, W, _ = bgr.shape
    out = np.empty_like(bgr)
    for k in range(F):
        for ch in range(3):
            g = EXP(-field_at_pixels(C[k, ch], W, H, spacing))
            v = bgr[k, :, :, ch].astype(f64) * g
            out[k, :, :, ch] = np.rint(np.minimum(np.maximum(v, 0.0), 255.0)).astype(np.uint8)
    return out


def true_log_gains(scene, seed=7):
    """log of scene.make_color_frames' gain fields [F, H, W, 3] (B, G, R), from the same RNG sequence."""
    F, H, W = np.asarray(scene["lum"]).shape
    rng = np.random.default_rng(seed)
    xx = np.arange(W, dtype=f64)[None, :]
    yy = np.arange(H, dtype=f64)[:, None]
    out = np.empty((F, H, W, 3))
    for f in range(F):
        ph = rng.uniform(0, 2 * np.pi, 3).astype(f32).astype(f64)
        out[f, :, :, 0] = np.log(0.85 + 0.07 * np.sin((xx + yy) / 53.0 + ph[2]))
        out[f, :, :, 1] = np.log(0.92 + 0.05 * np.cos(yy / 29.0 + ph[1])) + 0 * xx
        out[f, :, :, 2] = np.log(1.00 + 0.06 * np.sin(xx / 37.0 + ph[0])) + 0 * yy
    return out


def field_error(C, truth, mask, spacing):
    """RMS over the masked pixels [F, H, W] of l - log g_true - the channel's best constant, pooled over the channels."""
    F, H, W = mask.shape
    err = []
    for ch in range(3):
        d = np.concatenate([(field_at_pixels(C[k, ch], W, H, spacing) - truth[k, :, :, ch])[mask[k]] for k in range(F)])
        err.append(d - d.mean())
    e = np.concatenate(err)
    return float(np.sqrt((e * e).mean()))
