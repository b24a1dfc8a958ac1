"""numpy float32 restatement of the rasterizer of the resident mesh (intrinsic3d_b200/csrc/i3d_raster.cuh, DESIGN.md §6w).

Shares no code with the kernels.  Every float operation is one numpy float32 operation (IEEE round to nearest, no contraction), in the
order the kernel header states, so the planes and the integer statistics are byte-equal to the device's; the depth sums are float64 in
numpy's order (equal to the device's fixed-order sums to ~1e-15 relative).

Per pixel: the ray (x, y, 1) of render_ref's pixel rule; per face the camera-space vertices ((R0 p0 + R1 p1) + R2 p2) + t; the watertight
test of Woop, Benthin & Wald (2013) with the double recomputation of the edge functions when one is exactly 0; the winner is the
lexicographic minimum of (t, face); a face with every camera z <= 0 never hits.  The candidate pairs come from each face's padded box of
(X / Z, Y / Z) against the rays (all pixels for a face with a camera z <= 0 or a box that is not finite); brute=True tests every face
against every pixel instead.
"""
from __future__ import annotations

import numpy as np

import render_ref as rr
import texture_ref as tr

f32 = np.float32
PLANES = ("depth", "face", "bary", "normal", "rgb")
PAD = 2.0 ** -10            # the restatement's own box pad (relative to 1 + M + E); any pad at least the kernel's gives the same bytes


def rays(cam, W, H):
    """(x, y) float32 [H, W] of every pixel: (u - cx) / fx, (v - cy) / fy, then render_ref's fixed-point undistortion."""
    vv, uu = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    xd = (uu.astype(f32) - f32(cam["cx"])) / f32(cam["fx"])
    yd = (vv.astype(f32) - f32(cam["cy"])) / f32(cam["fy"])
    d = np.asarray(cam["d"], f32)
    if np.any(d != 0):
        with np.errstate(all="ignore"):
            xd, yd = rr._undistort(xd.astype(f32), yd.astype(f32), d)
    return xd.astype(f32), yd.astype(f32)


def camera_vertices(V, rt):
    """((R[k][0] p0 + R[k][1] p1) + R[k][2] p2) + t[k] for every vertex, float32 [V, 3]."""
    R, t = rt[:9].reshape(3, 3).astype(f32), rt[9:].astype(f32)
    return np.stack([((R[k, 0] * V[:, 0] + R[k, 1] * V[:, 1]) + R[k, 2] * V[:, 2]) + t[k] for k in range(3)], 1).astype(f32)


def hit(q, x, y):
    """The watertight test of rays (x, y, 1) [m] against camera-space triangles q [m, 3 vertices, 3]: (hit, t, a, b)."""
    m = len(x)
    ax, ay = np.abs(x), np.abs(y)
    kz = np.where(ax > ay, np.where(ax > 1, 0, 2), np.where(ay > 1, 1, 2))
    kx = (kz + 1) % 3
    ky = (kx + 1) % 3
    d = np.stack([x, y, np.ones(m, f32)], 1).astype(f32)
    take = lambda a, k: np.take_along_axis(a, k[:, None], 1)[:, 0]
    dz = take(d, kz)
    sw = dz < 0
    kx, ky = np.where(sw, ky, kx), np.where(sw, kx, ky)
    with np.errstate(all="ignore"):
        Sx, Sy, Sz = take(d, kx) / dz, take(d, ky) / dz, f32(1) / dz
        px, py, pz = [], [], []
        for j in range(3):
            zk = take(q[:, j], kz)
            px.append(take(q[:, j], kx) - Sx * zk)
            py.append(take(q[:, j], ky) - Sy * zk)
            pz.append(Sz * zk)
        U = px[2] * py[1] - py[2] * px[1]
        V = px[0] * py[2] - py[0] * px[2]
        W = px[1] * py[0] - py[1] * px[0]
        z0 = (U == 0) | (V == 0) | (W == 0)
        if z0.any():
            P = [(a.astype(np.float64), b.astype(np.float64)) for a, b in zip(px, py)]
            (Ax, Ay), (Bx, By), (Cx, Cy) = P
            U = np.where(z0, (Cx * By - Cy * Bx).astype(f32), U)
            V = np.where(z0, (Ax * Cy - Ay * Cx).astype(f32), V)
            W = np.where(z0, (Bx * Ay - By * Ax).astype(f32), W)
        ok = ~(((U < 0) | (V < 0) | (W < 0)) & ((U > 0) | (V > 0) | (W > 0)))
        det = (U + V) + W
        ok &= det != 0
        T = (U * pz[0] + V * pz[1]) + W * pz[2]
        t = T / det
        ok &= t > 0
        ok &= ~np.all(q[:, :, 2] <= 0, 1)                    # a face with every camera z <= 0 is a miss
        a, b = V / det, W / det
    return ok, t.astype(f32), a.astype(f32), b.astype(f32)


def _pairs(qv, Fc, rx, ry, brute):
    """Candidate (face, pixel) pairs of one view: faces with every z <= 0 dropped; every pixel for brute, a camera z <= 0 or a box
    that is not finite; else the pixels whose ray lies in the face's padded box."""
    H, W = rx.shape
    q = qv[Fc]                                           # [F, 3, 3]
    z = q[:, :, 2]
    behind = np.all(z <= 0, 1)
    front = np.all(z > 0, 1)
    with np.errstate(all="ignore"):
        X, Y = q[:, :, 0] / q[:, :, 2], q[:, :, 1] / q[:, :, 2]
        lo = np.stack([X.min(1), Y.min(1)], 1).astype(np.float64)
        hi = np.stack([X.max(1), Y.max(1)], 1).astype(np.float64)
        M = np.abs(np.concatenate([lo, hi], 1)).max(1)
        E = (hi - lo).max(1)
        pad = (1 + M + E) * PAD
        lo, hi = lo - pad[:, None], hi + pad[:, None]
    boxed = front & np.all(np.isfinite(lo), 1) & np.all(np.isfinite(hi), 1) & (not brute)
    faces, pix = [], []
    everything = np.nonzero(~boxed & (~behind | brute))[0]
    npx = H * W
    for c in range(0, len(everything), max(1, (1 << 22) // npx)):
        f = everything[c:c + max(1, (1 << 22) // npx)]
        faces.append(np.repeat(f, npx))
        pix.append(np.tile(np.arange(npx), len(f)))
    bf = np.nonzero(boxed)[0]
    if len(bf):
        # pixel rectangles from the rows' and columns' ray ranges (monotone envelopes, as conservative as the kernel's bands)
        rlo = np.minimum.accumulate(np.nanmin(ry, 1)[::-1])[::-1]
        rhi = np.maximum.accumulate(np.nanmax(ry, 1))
        clo = np.minimum.accumulate(np.nanmin(rx, 0)[::-1])[::-1]
        chi = np.maximum.accumulate(np.nanmax(rx, 0))
        r0 = np.searchsorted(rhi, lo[bf, 1], side="left")
        r1 = np.searchsorted(rlo, hi[bf, 1], side="right") - 1
        c0 = np.searchsorted(chi, lo[bf, 0], side="left")
        c1 = np.searchsorted(clo, hi[bf, 0], side="right") - 1
        nr, nc = np.maximum(r1 - r0 + 1, 0), np.maximum(c1 - c0 + 1, 0)
        cnt = nr * nc
        f = np.repeat(bf, cnt)
        k = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        ncr = np.repeat(nc, cnt)
        r = np.repeat(r0, cnt) + k // np.maximum(ncr, 1)
        cc = np.repeat(c0, cnt) + k % np.maximum(ncr, 1)
        p = r * W + cc
        x, y = rx.ravel()[p], ry.ravel()[p]
        inside = (x >= lo[f, 0]) & (x <= hi[f, 0]) & (y >= lo[f, 1]) & (y <= hi[f, 1])
        faces.append(f[inside])
        pix.append(p[inside])
    if not faces:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(faces).astype(np.int64), np.concatenate(pix).astype(np.int64)


def _texture_colour(face, a, b, image, S, cols, check_owned=True):
    """The atlas lookup of hits (face, a, b): R, G, B uint8 [m, 3]; asserts that every tap with weight > 0 is a texel the face owns."""
    ac, bc = np.where(a < 0, f32(0), a), np.where(b < 0, f32(0), b)
    s = (ac + bc).astype(f32)
    big = s > 1
    with np.errstate(all="ignore"):
        ac = np.where(big, ac / s, ac).astype(f32)
        bc = np.where(big, bc / s, bc).astype(f32)
    w = ((f32(1) - ac) - bc).astype(f32)
    fb = (face & 1).astype(bool)
    cu = np.where(fb[:, None, None], tr.uv_corners(S, True)[None], tr.uv_corners(S, False)[None])     # [m, 3, 2]
    u = ((w * cu[:, 0, 0] + ac * cu[:, 1, 0]) + bc * cu[:, 2, 0]).astype(f32)
    v = ((w * cu[:, 0, 1] + ac * cu[:, 1, 1]) + bc * cu[:, 2, 1]).astype(f32)
    cell = face // 2
    x0 = ((cell % cols) * S).astype(f32)
    y0 = ((cell // cols) * S).astype(f32)
    X = ((x0 + u) - f32(0.5)).astype(f32)
    Y = ((y0 + v) - f32(0.5)).astype(f32)
    if check_owned:
        fx, fy = np.floor(X), np.floor(Y)
        wx1, wy1 = X - fx, Y - fy
        for di, wx in ((0, 1 - wx1), (1, wx1)):
            for dj, wy in ((0, 1 - wy1), (1, wy1)):
                live = (wx * wy) > 0
                i = fx.astype(np.int64) + di - (cell % cols) * S
                j = fy.astype(np.int64) + dj - (cell // cols) * S
                own = np.where(fb, (i + j + 1 > S), (i + j + 1 < S)) & (i >= 0) & (i < S) & (j >= 0) & (j < S)
                assert np.all(own[live]), "a texture lookup read a texel its face does not own"
    return np.stack([tr.interp_u8(image, X, Y, k) for k in range(3)], 1)


def rasterize(mesh, rts, cam, W, H, color=None, texture=None, depth=None, bgr=None, ids=None, brute=False):
    """The planes [n, H, W] of every view (rts [n, 12] float32 world -> camera; with ids, view i uses rts[ids[i]] and frame ids[i]) and,
    with depth frames [F, H, W] (and bgr frames [F, H, W, 3] for the colour pairs), the per-view statistics.  color: None, "vertex" or
    "texture" with texture = (atlas image [h, w, 3] R, G, B, S)."""
    Vp = np.asarray(mesh["vertices"], f32).reshape(-1, 3)
    Fc = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    vcol = np.asarray(mesh["colors"], np.uint8).reshape(-1, 3)
    rts = np.asarray(rts, f32)
    views = list(ids) if ids is not None else list(range(len(rts)))
    n = len(views)
    rx, ry = rays(cam, W, H)
    nrm_f = tr.face_normals(Vp, Fc)
    out = dict(depth=np.zeros((n, H, W), f32), face=np.full((n, H, W), -1, np.int32), bary=np.zeros((n, H, W, 2), f32),
               normal=np.zeros((n, H, W, 3), f32), rgb=np.zeros((n, H, W, 3), np.uint8), stats=[], tests=0)
    if color == "texture":
        image, S = texture
        cols = tr.layout(len(Fc), S)["cols"]
    for i, vi in enumerate(views):
        qv = camera_vertices(Vp, rts[vi])
        f, p = _pairs(qv, Fc, rx, ry, brute)
        out["tests"] += len(f)
        ok, t, a, b = hit(qv[Fc[f]], rx.ravel()[p], ry.ravel()[p])
        f, p, t, a, b = f[ok], p[ok], t[ok], a[ok], b[ok]
        order = np.lexsort((f, t, p))                     # by pixel, then t, then face
        f, p, t, a, b = f[order], p[order], t[order], a[order], b[order]
        first = np.ones(len(p), bool)
        first[1:] = p[1:] != p[:-1]
        f, p, t, a, b = f[first], p[first], t[first], a[first], b[first]
        dep, fac, bar, nor, rgb = (out[k][i].reshape(H * W, *out[k].shape[3:]) for k in PLANES)
        dep[p], fac[p], bar[p, 0], bar[p, 1], nor[p] = t, f, a, b, nrm_f[f]
        if color == "vertex":
            w0 = ((f32(1) - a) - b).astype(f32)
            c = Fc[f]
            x = (((w0[:, None] * vcol[c[:, 0]].astype(f32) + a[:, None] * vcol[c[:, 1]].astype(f32)) + b[:, None] * vcol[c[:, 2]].astype(f32))
                 + f32(0.5)).astype(f32)
            rgb[p] = np.trunc(np.clip(x, f32(0), f32(255))).astype(np.uint8)
        elif color == "texture":
            rgb[p] = _texture_colour(f, a, b, image, S, cols)
        if depth is not None:
            zo = np.asarray(depth[vi], f32).reshape(-1)
            cov = np.zeros(H * W, bool)
            cov[p] = True
            obs = zo > 0
            dp = cov & obs
            e = dep[dp].astype(np.float64) - zo[dp].astype(np.float64)
            st = dict(num_covered=int(cov.sum()), num_observed=int(obs.sum()), depth_count=int(dp.sum()), color_count=0,
                      depth_abs=float(np.abs(e).sum()), depth_sq=float((e * e).sum()), color_abs=[0, 0, 0], color_sq=[0, 0, 0])
            if color is not None and bgr is not None:
                fr = np.asarray(bgr[vi], np.uint8).reshape(-1, 3)
                ec = rgb[cov].astype(np.int64) - fr[cov][:, ::-1].astype(np.int64)
                st["color_count"] = int(cov.sum())
                st["color_abs"] = [int(v) for v in np.abs(ec).sum(0)]
                st["color_sq"] = [int(v) for v in (ec * ec).sum(0)]
            out["stats"].append(st)
    return out
