"""numpy restatement of frame-to-model tracking (intrinsic3d_b200/csrc/i3d_track.cuh, DESIGN.md §6n).

The prediction is tests/render_ref.py's dense march (geometry only) at the input pose; the depth pyramid is tests/frames_ref.py's
depth_down chain.  Every float operation is one numpy float32 operation and every double operation one float64 operation (IEEE round to
nearest, no contraction), in the device's order, so the pyramid, normals, prediction planes and correspondence masks are byte-equal and
the per-frame sums are the device's bit for bit (warp shuffle tree, warps in order, tiles in order).  The solve is restated in Python
floats; its only libm calls are sin and cos of the update angle, so poses after an update agree to the last bits, not bit for bit.
"""
from __future__ import annotations

import math

import numpy as np

import frames_ref
import render_ref as rr

f32 = np.float32
VALS = 29                 # kTrackVals: 21 upper-triangle entries of J^T J, 6 of J^T r, r^2, rows
TILE = 16                 # kTrackTile
UPPER = [(a, b) for a in range(6) for b in range(a, 6)]
DEFAULTS = dict(num_levels=3, iterations=(10, 5, 4, 0), max_distance=0.05, min_normal_cos=math.cos(math.radians(20.0)),
                min_correspondences=100)


def params(**over):
    p = dict(DEFAULTS)
    p.update(over)
    it = list(p["iterations"]) + [0] * (4 - len(p["iterations"]))
    p["iterations"] = tuple(int(x) for x in it)
    p["max_distance"] = f32(p["max_distance"])
    p["min_normal_cos"] = f32(p["min_normal_cos"])
    return p


def level_cams(dcam, levels):
    """The depth camera (W, H, fx, fy, cx, cy) at levels 0..levels-1: sizes halved (floor), intrinsics * 2^-l in float."""
    W, H, fx, fy, cx, cy = dcam
    out = []
    for l in range(levels):
        s = 2.0 ** -l
        out.append(dict(W=int(W), H=int(H), fx=f32(float(f32(fx)) * s), fy=f32(float(f32(fy)) * s), cx=f32(float(f32(cx)) * s),
                        cy=f32(float(f32(cy)) * s)))
        W, H = W // 2, H // 2
    return out


def pyramid(depth0, levels):
    """depth planes of levels 0..levels-1 of one frame (k_frames_depthdown chain)."""
    out = [np.asarray(depth0, f32)]
    for _ in range(1, levels):
        out.append(frames_ref.depth_down(out[-1]))
    return out


def normals(depth, cam):
    """camera-frame normals [H, W, 3] by the computeNormals(K, depth, 0.3) rule of k_fuse_normals."""
    d = np.asarray(depth, f32)
    H, W = d.shape
    out = np.zeros((H, W, 3), f32)
    if H < 3 or W < 3:
        return out
    fxi, fyi = f32(1.0) / cam["fx"], f32(1.0) / cam["fy"]
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")

    def vert(dy, dx):
        y, x = ys[1:-1, 1:-1] + dy, xs[1:-1, 1:-1] + dx
        dd = d[y, x]
        return ((x.astype(f32) - cam["cx"]) * fxi) * dd, ((y.astype(f32) - cam["cy"]) * fyi) * dd, dd
    vx0, vx1, vy0, vy1 = vert(0, -1), vert(0, 1), vert(-1, 0), vert(1, 0)
    tx = [vx1[k] - vx0[k] for k in range(3)]
    ty = [vy1[k] - vy0[k] for k in range(3)]
    lx = np.sqrt((tx[0] * tx[0] + tx[1] * tx[1]) + tx[2] * tx[2])
    ly = np.sqrt((ty[0] * ty[0] + ty[1] * ty[1]) + ty[2] * ty[2])
    ok = (d[1:-1, 1:-1] != 0) & (vx0[2] != 0) & (vx1[2] != 0) & (vy0[2] != 0) & (vy1[2] != 0) & (lx < f32(0.3)) & (ly < f32(0.3))
    c = [ty[1] * tx[2] - ty[2] * tx[1], ty[2] * tx[0] - ty[0] * tx[2], ty[0] * tx[1] - ty[1] * tx[0]]
    sq = (c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]
    pos = sq > 0
    ln = np.sqrt(np.where(pos, sq, f32(1.0)))
    inner = np.stack([np.where(pos, ck / ln, ck) for ck in c], -1)
    out[1:-1, 1:-1] = np.where(ok[..., None], inner, f32(0.0))
    return out


def xform(R, t, v):
    """R (row-major [12] or [9]) times v (list of 3 arrays), sums left to right, plus t when given."""
    out = []
    for d in range(3):
        s = (R[3 * d] * v[0] + R[3 * d + 1] * v[1]) + R[3 * d + 2] * v[2]
        out.append(s + t[d] if t is not None else s)
    return out


def predict(grid, rt_in, cam0, depth_obs):
    """The prediction at the input pose rt_in (float world -> camera [12]): (depth [H, W], normal [H, W, 3], initial stats)."""
    cam = dict(fx=cam0["fx"], fy=cam0["fy"], cx=cam0["cx"], cy=cam0["cy"], d=np.zeros(5, f32))
    view = rr.render_view(grid, np.asarray(rt_in, f32), cam, cam0["W"], cam0["H"], photometric=False)
    st = rr.stats(view, np.asarray(depth_obs, f32), np.zeros_like(depth_obs, dtype=f32))
    return view["depth"], view["normal"], st


def associate(depth, nrm, cam, Tf, rt_in, cam0, pdepth, pnrm, p):
    """Correspondences of every pixel of one level at the float pose Tf (camera -> world [12]): (ok [H, W], p, q, n_m as [3] lists of
    [H, W] float32 arrays; meaningful where ok)."""
    H, W = depth.shape
    vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    u, v = uu.astype(f32), vv.astype(f32)
    z = depth
    ok = z > 0
    vc = [((u - cam["cx"]) / cam["fx"]) * z, ((v - cam["cy"]) / cam["fy"]) * z, z]
    Tf = np.asarray(Tf, f32)
    R0 = np.asarray(rt_in, f32)
    with np.errstate(all="ignore"):
        pw = xform(Tf, Tf[9:], vc)
        pc = xform(R0, R0[9:], pw)
        ok &= pc[2] > 0
        tu = ((cam0["fx"] * (pc[0] / pc[2])) + cam0["cx"]) + f32(0.5)
        tv = ((cam0["fy"] * (pc[1] / pc[2])) + cam0["cy"]) + f32(0.5)
        ok &= (tu > f32(-1.0)) & (tu < f32(cam0["W"])) & (tv > f32(-1.0)) & (tv < f32(cam0["H"]))
        iu = np.where(ok, np.trunc(np.where(ok, tu, 0)), 0).astype(np.int64)
        iv = np.where(ok, np.trunc(np.where(ok, tv, 0)), 0).astype(np.int64)
        zm = pdepth[iv, iu]
        ok &= zm > 0
        nm = [pnrm[iv, iu, k] for k in range(3)]
        ok &= ~((nm[0] == 0) & (nm[1] == 0) & (nm[2] == 0))
        xn = (iu.astype(f32) - cam0["cx"]) / cam0["fx"]
        yn = (iv.astype(f32) - cam0["cy"]) / cam0["fy"]
        q = []
        dsq = np.zeros((H, W), f32)
        for k in range(3):
            o = -((R0[k] * R0[9] + R0[3 + k] * R0[10]) + R0[6 + k] * R0[11])
            dr = (R0[k] * xn + R0[3 + k] * yn) + R0[6 + k]
            q.append(o + zm * dr)
            e = pw[k] - q[k]
            dsq = dsq + e * e
        ok &= dsq <= p["max_distance"] * p["max_distance"]
        if p["min_normal_cos"] > f32(-1.0):
            nin = xform(Tf, None, [nrm[..., 0], nrm[..., 1], nrm[..., 2]])
            dot = (nin[0] * nm[0] + nin[1] * nm[1]) + nin[2] * nm[2]
            ok &= dot >= p["min_normal_cos"]
    return ok, pw, q, nm


def rows(ok, pw, q, nm):
    """The point-to-plane rows in double: J [H, W, 6], r [H, W] (0 where there is no correspondence)."""
    pd = [np.where(ok, pw[k], 0).astype(np.float64) for k in range(3)]
    qd = [np.where(ok, q[k], 0).astype(np.float64) for k in range(3)]
    nd = [np.where(ok, nm[k], 0).astype(np.float64) for k in range(3)]
    r = (nd[0] * (pd[0] - qd[0]) + nd[1] * (pd[1] - qd[1])) + nd[2] * (pd[2] - qd[2])
    J = np.stack([pd[1] * nd[2] - pd[2] * nd[1], pd[2] * nd[0] - pd[0] * nd[2], pd[0] * nd[1] - pd[1] * nd[0], nd[0], nd[1], nd[2]], -1)
    return J, r


def values(J, r, ok):
    """the 29 per-pixel values [H, W, 29]"""
    H, W = r.shape
    V = np.empty((H, W, VALS), np.float64)
    for j, (a, b) in enumerate(UPPER):
        V[..., j] = J[..., a] * J[..., b]
    for a in range(6):
        V[..., 21 + a] = J[..., a] * r
    V[..., 27] = r * r
    V[..., 28] = ok.astype(np.float64)
    return V


def tile_sums(V):
    """the device's order: per 16 x 16 tile a shuffle tree over each warp (2 rows), the 8 warps in order, then the tiles in order"""
    H, W, _ = V.shape
    ty, tx = -(-H // TILE), -(-W // TILE)
    P = np.zeros((ty * TILE, tx * TILE, VALS), np.float64)
    P[:H, :W] = V
    x = P.reshape(ty, TILE, tx, TILE, VALS).transpose(0, 2, 1, 3, 4).reshape(ty, tx, 8, 32, VALS).copy()
    for o in (16, 8, 4, 2, 1):
        x[:, :, :, :o] = x[:, :, :, :o] + x[:, :, :, o:2 * o]
    w = x[:, :, :, 0]
    t = w[:, :, 0]
    for k in range(1, 8):
        t = t + w[:, :, k]
    t = t.reshape(ty * tx, VALS)
    s = np.zeros(VALS, np.float64)
    for k in range(ty * tx):
        s = s + t[k]
    return s


def inverse(T):
    """R^T | -(R^T t) of R | t (row-major [12]) in double, sums left to right"""
    T = [float(a) for a in T]
    out = [0.0] * 12
    for i in range(3):
        for j in range(3):
            out[3 * i + j] = T[3 * j + i]
        out[9 + i] = -((T[i] * T[9] + T[3 + i] * T[10]) + T[6 + i] * T[11])
    return out


def rodrigues(w):
    th2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
    th = math.sqrt(th2)
    R = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    if th > 0.0:
        sa, sb = math.sin(th) / th, (1.0 - math.cos(th)) / th2
        K = [0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0]
        for a in range(3):
            for c in range(3):
                k2 = (K[3 * a] * K[c] + K[3 * a + 1] * K[3 + c]) + K[3 * a + 2] * K[6 + c]
                R[3 * a + c] = (R[3 * a + c] + sa * K[3 * a + c]) + sb * k2
    return R


def solve(S):
    """(status, xi): Cholesky of the 6 x 6 system in the device's order and xi = -A^-1 b; status 2 (not positive definite) or 3
    (non-finite) without xi"""
    S = [float(a) for a in S]
    if not all(math.isfinite(a) for a in S):
        return 3, None
    A = [[0.0] * 6 for _ in range(6)]
    for j, (a, b) in enumerate(UPPER):
        A[a][b] = A[b][a] = S[j]
    b = S[21:27]
    L = [[0.0] * 6 for _ in range(6)]
    for c in range(6):
        d = A[c][c]
        for m in range(c):
            d = d - L[c][m] * L[c][m]
        if not d > 0.0:
            return 2, None
        L[c][c] = math.sqrt(d)
        for i in range(c + 1, 6):
            t = A[i][c]
            for m in range(c):
                t = t - L[i][m] * L[c][m]
            L[i][c] = t / L[c][c]
    y = [0.0] * 6
    for i in range(6):
        t = -b[i]
        for m in range(i):
            t = t - L[i][m] * y[m]
        y[i] = t / L[i][i]
    x = [0.0] * 6
    for i in range(5, -1, -1):
        t = y[i]
        for m in range(i + 1, 6):
            t = t - L[m][i] * x[m]
        x[i] = t / L[i][i]
    return 0, x


def update(T, x):
    """[Rodrigues(w) | v] . T (camera -> world), in double"""
    R = rodrigues(x[:3])
    out = [0.0] * 12
    for a in range(3):
        for c in range(3):
            out[3 * a + c] = (R[3 * a] * T[c] + R[3 * a + 1] * T[3 + c]) + R[3 * a + 2] * T[6 + c]
        out[9 + a] = ((R[3 * a] * T[9] + R[3 * a + 1] * T[10]) + R[3 * a + 2] * T[11]) + x[3 + a]
    return out


class Frame:
    """One frame's tracking problem: its pyramid with normals, the prediction at the input pose and the schedule's state."""

    def __init__(self, depth0, pose_in, dcam, p, grid=None, prediction=None):
        self.p = p
        self.cams = level_cams(dcam, p["num_levels"])
        self.depth = pyramid(depth0, p["num_levels"])
        self.nrm = [normals(d, c) for d, c in zip(self.depth, self.cams)]
        self.pose_in = np.asarray(pose_in, np.float64)
        self.rt_in = self.pose_in.astype(f32)
        if prediction is None:
            self.pdepth, self.pnrm, self.initial = predict(grid, self.rt_in, self.cams[0], self.depth[0])
        else:
            self.pdepth, self.pnrm = (np.asarray(a, f32) for a in prediction)
            self.initial = None
        self.T = inverse(self.pose_in)
        self.w2c = [float(a) for a in self.pose_in]
        self.status, self.iterations, self.frozen = 0, 0, False
        self.correspondences, self.residual_sq, self.update_norm = 0, 0.0, 0.0
        self.sys = np.zeros(VALS)
        self.mask = np.zeros(self.depth[0].shape, np.uint8)

    def Tf(self):
        return np.asarray(self.T, np.float64).astype(f32)

    def system(self, l):
        ok, pw, q, nm = associate(self.depth[l], self.nrm[l], self.cams[l], self.Tf(), self.rt_in, self.cams[0], self.pdepth, self.pnrm, self.p)
        if l == 0:
            self.mask = ok.astype(np.uint8)
        J, r = rows(ok, pw, q, nm)
        return tile_sums(values(J, r, ok))

    def step(self, l, do_solve=True):
        """one k_track_rows / k_track_finish / k_track_solve of this frame"""
        if self.frozen:
            return
        S = self.system(l)
        self.sys = S
        self.correspondences, self.residual_sq = int(S[28]), float(S[27])
        if not do_solve:
            return
        if self.correspondences < self.p["min_correspondences"]:
            self.status, self.frozen = 1, True
            return
        status, x = solve(S)
        if status:
            self.status, self.frozen = status, True
            return
        T = update(self.T, x)
        if not all(math.isfinite(a) for a in list(x) + T):
            self.status, self.frozen = 3, True
            return
        self.T = T
        self.w2c = inverse(T)
        self.update_norm = math.sqrt(sum_sq(x))
        self.iterations += 1

    def run(self):
        it = self.p["iterations"]
        for l in range(self.p["num_levels"] - 1, -1, -1):
            for _ in range(it[l]):
                self.step(l)
        if sum(it[:self.p["num_levels"]]) == 0:
            self.step(0, do_solve=False)
        return self


def sum_sq(x):
    s = 0.0
    for a in x:
        s = s + a * a
    return s


def track(grid, depth_frames, ids, pose_in, dcam, **over):
    """i3d_track_sensor_frames restated: one Frame per id (run), in call order."""
    p = params(**over)
    return [Frame(depth_frames[f], pose_in[k], dcam, p, grid=grid).run() for k, f in enumerate(ids)]


# ---- poses ------------------------------------------------------------------------------------------------------------------------
def aa_to_rt(poses):
    """angle-axis + translation [F, 6] (world -> camera) -> R row-major | t [F, 12] in double"""
    from intrinsic3d_b200.scene import aa_to_rotation
    out = np.zeros((len(poses), 12))
    for f, p in enumerate(np.asarray(poses, np.float64)):
        out[f, :9] = aa_to_rotation(p[:3]).reshape(-1)
        out[f, 9:] = p[3:]
    return out


def pose_errors(est, true):
    """(rotation error in degrees, camera-centre error in metres) of world -> camera poses [n, 12] against the truth"""
    est, true = np.asarray(est, np.float64), np.asarray(true, np.float64)
    rot, trans = [], []
    for a, b in zip(est, true):
        Ra, Rb = a[:9].reshape(3, 3), b[:9].reshape(3, 3)
        c = (np.trace(Ra @ Rb.T) - 1.0) * 0.5
        rot.append(math.degrees(math.acos(min(1.0, max(-1.0, c)))))
        trans.append(float(np.linalg.norm(Ra.T @ a[9:] - Rb.T @ b[9:])))
    return np.array(rot), np.array(trans)


def perturb(rt, rot_deg, trans_m, seed):
    """world -> camera poses [n, 12] with each camera rotated by rot_deg about a random axis and moved by trans_m in a random direction"""
    from intrinsic3d_b200.scene import aa_to_rotation
    rng = np.random.default_rng(seed)
    out = np.array(rt, np.float64)
    for f in range(len(out)):
        a = rng.normal(size=3); a /= np.linalg.norm(a)
        d = rng.normal(size=3); d /= np.linalg.norm(d)
        R = out[f, :9].reshape(3, 3)
        c = -R.T @ out[f, 9:] + trans_m * d
        Rn = aa_to_rotation(a * math.radians(rot_deg)) @ R
        out[f, :9] = Rn.reshape(-1)
        out[f, 9:] = -Rn @ c
    return out
