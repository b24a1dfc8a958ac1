"""numpy float32 restatement of the keyframe renderer (intrinsic3d_b200/csrc/i3d_render.cuh, DESIGN.md §6m).

Shares no code with the kernels: neighbours come from a sorted key table of the voxel coordinates (np.searchsorted), not from the
engine's neighbour table, and only the dense march is restated (every lattice sample is evaluated; the device's empty-space skipping
must not change a result).  Every float operation is one numpy float32 operation (IEEE round to nearest, no contraction), so the planes
are byte-equal to the device's; the statistics are float64 sums in numpy's order (equal to the device's to ~1e-15 relative).
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32
UNDISTORT_ITERS = 10          # kUndistortIters of i3d_render.h
MAX_LATTICE = 1 << 24         # kRenderMaxLattice: the last lattice index a ray may sample
PLANES = ("depth", "normal", "albedo", "shading", "intensity")


def pose_rt(poses):
    """k_pose_mats: math::poseVecAAToMat in float64, cast to float: [F, 12] = R row-major | t (world -> camera)."""
    poses = np.asarray(poses, np.float64)
    out = np.zeros((len(poses), 12), f32)
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
        out[f, :9] = np.array(M, np.float64).astype(f32)
        out[f, 9:] = p[3:].astype(f32)
    return out


def camera(intr, dist, pyr_scale=1.0):
    """select_cam: intrinsics * pyr_scale and the distortion, cast to float."""
    fx, fy, cx, cy = (f32(float(a) * float(pyr_scale)) for a in intr)
    return dict(fx=fx, fy=fy, cx=cx, cy=cy, d=np.asarray(dist, np.float64).astype(f32))


class KeyTable:
    """Voxel coordinates -> index through a sorted table of packed keys."""

    def __init__(self, xyz):
        xyz = np.asarray(xyz, np.int64)
        k = self.pack(xyz[:, 0], xyz[:, 1], xyz[:, 2])
        self.order = np.argsort(k, kind="stable")
        self.keys = k[self.order]

    @staticmethod
    def pack(x, y, z):
        b = 1 << 20
        return ((x + b) << 42) | ((y + b) << 21) | (z + b)

    def find(self, x, y, z):
        k = self.pack(x, y, z)
        pos = np.minimum(np.searchsorted(self.keys, k), len(self.keys) - 1)
        return np.where(self.keys[pos] == k, self.order[pos], -1)


def lerp(a, b, t):
    return a + t * (b - a)


def _undistort(xd, yd, d):
    x, y = xd, yd
    two = f32(2.0)
    for _ in range(UNDISTORT_ITERS):
        r2 = x * x + y * y
        r4 = r2 * r2
        r6 = r4 * r2
        dc = ((f32(1.0) + d[0] * r2) + d[1] * r4) + d[2] * r6
        tx = ((two * d[3]) * x) * y + d[4] * (r2 + (two * x) * x)
        ty = ((two * d[4]) * xd) * y + d[3] * (r2 + (two * y) * y)
        x = (xd - tx) / dc
        y = (yd - ty) / dc
    return x, y


def project(p, rt, cam):
    """observation_weight's forward projection of world points p [m, 3] -> (pu, pv) (round-trip checks)."""
    R, t = rt[:9].reshape(3, 3), rt[9:]
    q = [((R[k, 0] * p[:, 0] + R[k, 1] * p[:, 1]) + R[k, 2] * p[:, 2]) + t[k] for k in range(3)]
    x, y = q[0] / q[2], q[1] / q[2]
    d = cam["d"]
    if np.any(d != 0):
        two = f32(2.0)
        r2 = x * x + y * y
        r4 = r2 * r2
        r6 = r4 * r2
        dc = ((f32(1.0) + d[0] * r2) + d[1] * r4) + d[2] * r6
        xn = (x * dc + ((two * d[3]) * x) * y) + d[4] * (r2 + (two * x) * x)
        yn = (y * dc + ((two * d[4]) * xn) * y) + d[3] * (r2 + (two * y) * y)
        x, y = xn, yn
    return cam["fx"] * x + cam["cx"], cam["fy"] * y + cam["cy"]


class Grid:
    """The voxel set as the march reads it: sdf (the source), albedo, weight as float arrays of the downloaded grid; sh [n, 9] and
    sh_has [n] (None without photometric outputs)."""

    def __init__(self, xyz, sdf, albedo, weight, voxel_size, sh=None, sh_has=None):
        self.xyz = np.asarray(xyz, np.int64)
        self.sdf = np.asarray(sdf, np.float64).astype(f32)
        self.albedo = np.asarray(albedo, np.float64).astype(f32)
        self.weight = np.asarray(weight, f32)
        self.vs = f32(voxel_size)
        self.sh = None if sh is None else np.asarray(sh, np.float64).astype(f32)
        self.sh_has = None if sh_has is None else np.asarray(sh_has) != 0
        self.table = KeyTable(self.xyz)
        self.lo = self.xyz.min(0).astype(f32) * self.vs
        self.hi = self.xyz.max(0).astype(f32) * self.vs

    def cube(self, p):
        """base voxel, fractions, corner ids [m, 8] (corner i = dx + 2 dy + 4 dz) and the cube rule (all exist with weight != 0)"""
        gd = p / self.vs
        fl = np.floor(gd)
        base = fl.astype(np.int64)
        f = gd - fl
        c = np.empty((len(p), 8), np.int64)
        for i in range(8):
            c[:, i] = self.table.find(base[:, 0] + (i & 1), base[:, 1] + ((i >> 1) & 1), base[:, 2] + ((i >> 2) & 1))
        ok = np.all(c >= 0, 1)
        ok &= np.all(self.weight[np.maximum(c, 0)] != 0, 1)
        return c, f, ok

    @staticmethod
    def trilinear(vals, c, f):
        s = vals[np.maximum(c, 0)]
        a00, a10 = lerp(s[:, 0], s[:, 1], f[:, 0]), lerp(s[:, 2], s[:, 3], f[:, 0])
        a01, a11 = lerp(s[:, 4], s[:, 5], f[:, 0]), lerp(s[:, 6], s[:, 7], f[:, 0])
        return lerp(lerp(a00, a10, f[:, 1]), lerp(a01, a11, f[:, 1]), f[:, 2])


def normals(s, f):
    a00, a10 = lerp(s[:, 0], s[:, 1], f[:, 0]), lerp(s[:, 2], s[:, 3], f[:, 0])
    a01, a11 = lerp(s[:, 4], s[:, 5], f[:, 0]), lerp(s[:, 6], s[:, 7], f[:, 0])
    b0, b1 = lerp(a00, a10, f[:, 1]), lerp(a01, a11, f[:, 1])
    gx = lerp(lerp(s[:, 1] - s[:, 0], s[:, 3] - s[:, 2], f[:, 1]), lerp(s[:, 5] - s[:, 4], s[:, 7] - s[:, 6], f[:, 1]), f[:, 2])
    gy = lerp(a10 - a00, a11 - a01, f[:, 2])
    gz = b1 - b0
    ln = np.sqrt((gx * gx + gy * gy) + gz * gz)
    nz = ln != 0
    safe = np.where(nz, ln, f32(1.0))
    n = np.stack([gx / safe, gy / safe, gz / safe], 1)
    n[~nz] = 0
    return n


def sh_blend(grid, c, f):
    """per-voxel SH of the corners, weights (wx * wy) * wz, renormalised over the corners with SH; (sh [m, 9], defined [m])"""
    m = len(c)
    acc = np.zeros((m, 9), f32)
    wsum = np.zeros(m, f32)
    for i in range(8):
        has = grid.sh_has[c[:, i]]
        wx = f[:, 0] if i & 1 else f32(1.0) - f[:, 0]
        wy = f[:, 1] if i & 2 else f32(1.0) - f[:, 1]
        wz = f[:, 2] if i & 4 else f32(1.0) - f[:, 2]
        w = (wx * wy) * wz
        for k in range(9):
            acc[:, k] = np.where(has, acc[:, k] + w * grid.sh[c[:, i], k], acc[:, k])
        wsum = np.where(has, wsum + w, wsum)
    ok = wsum > 0
    out = acc / np.where(ok, wsum, f32(1.0))[:, None]
    return out, ok


def shading(n, sh, albedo):
    """Shading::computeShading as i3d_vis.cuh's vis_shading restates it: albedo * (sh . basis(n)); 0 for albedo 0 or NaN"""
    x, y, z = n[:, 0], n[:, 1], n[:, 2]
    b = [np.ones_like(x), y, z, x, x * y, y * z, (-(x * x) - y * y) + f32(2.0) * (z * z), x * z, x * x - y * y]
    d = sh[:, 0] * b[0]
    for k in range(1, 9):
        d = d + sh[:, k] * b[k]
    out = albedo * d
    return np.where((albedo == 0) | np.isnan(albedo), f32(0.0), out)


def render_view(grid, rt, cam, W, H, photometric=True):
    """The planes of one view: depth [H, W], normal [H, W, 3], albedo, shading, intensity, shade_ok [H, W]."""
    rt = np.asarray(rt, f32)
    vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    u, v = uu.ravel().astype(f32), vv.ravel().astype(f32)
    xd = (u - cam["cx"]) / cam["fx"]
    yd = (v - cam["cy"]) / cam["fy"]
    x, y = (xd, yd) if not np.any(cam["d"] != 0) else _undistort(xd, yd, cam["d"])
    o = np.empty(3, f32)
    dn = np.empty((len(u), 3), f32)
    with np.errstate(invalid="ignore", over="ignore"):         # a non-finite pose gives a non-finite ray, which has no samples
        for d in range(3):
            o[d] = -((rt[d] * rt[9] + rt[3 + d] * rt[10]) + rt[6 + d] * rt[11])
            dn[:, d] = (rt[d] * x + rt[3 + d] * y) + rt[6 + d]
        ln = np.sqrt((dn[:, 0] * dn[:, 0] + dn[:, 1] * dn[:, 1]) + dn[:, 2] * dn[:, 2])
        dn = dn / ln[:, None]
    m = len(u)
    s0 = np.zeros(m, f32)
    s1 = np.full(m, np.inf, f32)
    any_ = np.ones(m, bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        for d in range(3):
            nz = dn[:, d] != 0
            ta = (grid.lo[d] - o[d]) / dn[:, d]
            tb = (grid.hi[d] - o[d]) / dn[:, d]
            s0 = np.where(nz, np.maximum(s0, np.minimum(ta, tb)), s0)
            s1 = np.where(nz, np.minimum(s1, np.maximum(ta, tb)), s1)
            any_ &= nz | ~((o[d] < grid.lo[d]) | (o[d] > grid.hi[d]))
    h = grid.vs * f32(0.5)
    # a non-finite ray (NaN or infinite pose) has no samples
    finite = np.isfinite(s1) & np.all(np.isfinite(dn), 1) & bool(np.all(np.isfinite(o)))
    active = any_ & finite & (s0 <= s1)
    k = np.zeros(m, np.int64)
    prev_ok = np.zeros(m, bool)
    prev = np.zeros(m, f32)
    hit = np.zeros(m, bool)
    s_hit = np.zeros(m, f32)
    hit_c = np.zeros((m, 8), np.int64)
    hit_f = np.zeros((m, 3), f32)
    while True:
        idx = np.nonzero(active)[0]
        if len(idx) == 0:
            break
        s = s0[idx] + k[idx].astype(f32) * h
        done = ~(s <= s1[idx]) | (k[idx] > MAX_LATTICE)
        active[idx[done]] = False
        idx, s = idx[~done], s[~done]
        p = o[None, :] + s[:, None] * dn[idx]
        c, f, ok = grid.cube(p)
        val = Grid.trilinear(grid.sdf, c, f)
        cross = ok & prev_ok[idx] & (prev[idx] > 0) & (val <= 0)
        if cross.any():
            ci = idx[cross]
            pv, cv = prev[ci], val[cross]
            tau = pv / (pv - cv)
            sc = (s0[ci] + (k[ci] - 1).astype(f32) * h) + tau * h
            pc = o[None, :] + sc[:, None] * dn[ci]
            cc, fc, okc = grid.cube(pc)
            hi_ = ci[okc]
            hit[hi_] = True
            s_hit[hi_] = sc[okc]
            hit_c[hi_] = cc[okc]
            hit_f[hi_] = fc[okc]
            active[hi_] = False
        prev_ok[idx] = ok
        prev[idx] = np.where(ok, val, prev[idx])
        k[idx] += 1
    depth = np.zeros(m, f32)
    nrm = np.zeros((m, 3), f32)
    alb = np.zeros(m, f32)
    shade = np.zeros(m, f32)
    inten = np.zeros(m, f32)
    shade_ok = np.zeros(m, bool)
    hi_ = np.nonzero(hit)[0]
    if len(hi_):
        c, f = hit_c[hi_], hit_f[hi_]
        depth[hi_] = s_hit[hi_] / ln[hi_]
        nrm[hi_] = normals(grid.sdf[c], f)
        alb[hi_] = Grid.trilinear(grid.albedo, c, f)
        if photometric:
            sh, ok = sh_blend(grid, c, f)
            ok &= ~np.all(nrm[hi_] == 0, 1)
            sel = hi_[ok]
            shade[sel] = shading(nrm[sel], sh[ok], np.ones(len(sel), f32))
            inten[sel] = shading(nrm[sel], sh[ok], alb[sel])
            shade_ok[sel] = True
    return dict(depth=depth.reshape(H, W), normal=nrm.reshape(H, W, 3), albedo=alb.reshape(H, W), shading=shade.reshape(H, W),
                intensity=inten.reshape(H, W), hit=hit.reshape(H, W), shade_ok=shade_ok.reshape(H, W), ray=(o, dn.reshape(H, W, 3)),
                s_hit=s_hit.reshape(H, W))


def stats(view, depth_obs, lum_obs):
    """I3DRenderStats of one view against its frame (float64 sums)."""
    hit, obs = view["hit"], np.asarray(depth_obs, f32) > 0
    dp = hit & obs
    dz = view["depth"][dp].astype(np.float64) - depth_obs[dp].astype(np.float64)
    pp = view["shade_ok"] & obs
    di = view["intensity"][pp].astype(np.float64) - lum_obs[pp].astype(np.float64)
    return dict(num_hit=int(hit.sum()), num_observed=int(obs.sum()), depth_count=int(dp.sum()), photo_count=int(pp.sum()),
                depth_abs=float(np.abs(dz).sum()), depth_sq=float((dz * dz).sum()), photo_abs=float(np.abs(di).sum()),
                photo_sq=float((di * di).sum()))


def render(grid, poses, intr, dist, pyr_scale, ids, depth_frames, lum_frames, photometric=True):
    """Every view of ids: planes [n, H, W] (normal [n, H, W, 3]) and the per-view statistics, as i3d_render_keyframes gives them."""
    rts = pose_rt(poses)
    cam = camera(intr, dist, pyr_scale)
    _, H, W = np.asarray(depth_frames).shape
    views = [render_view(grid, rts[f], cam, W, H, photometric) for f in ids]
    out = {p: np.stack([v[p] for v in views]) for p in PLANES}
    out["stats"] = [stats(v, depth_frames[f], lum_frames[f]) for v, f in zip(views, ids)]
    out["views"] = views
    return out


def grid_of(g, source, sh=None, sh_has=None):
    """Grid of a downloaded engine grid (Engine.download_grid) for source "fused" (sdf0) or "refined"."""
    sdf = g["sdf0"] if source == "fused" else g["sdf_refined"]
    return Grid(g["xyz"], sdf, g["albedo"], g["weight"], g["voxel_size"], sh, sh_has)
