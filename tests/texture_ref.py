"""numpy float32 restatement of the texture bake (intrinsic3d_b200/csrc/i3d_texture.cuh, DESIGN.md §6t).

Shares no code with the kernels.  Every float operation is one numpy float32 operation (IEEE round to nearest, no contraction), in the
order the kernel header states, so the atlas, the UVs and the counts are byte-equal to the device's.  The frame culling is not restated:
it only skips frames of weight exactly 0.

Layout: faces 2c and 2c+1 share cell c of S x S texels, cols = ceil(sqrt(ceil(F / 2))), rows = ceil(ncells / cols); local texel (i, j)
has its centre at (i + 1/2, j + 1/2), v down.  Face A = 2c has UV corners (1, 1), (S-3, 1), (1, S-3) and owns i + j + 1 < S; face B = 2c+1
has (S-1, S-1), (3, S-1), (S-1, 3) and owns i + j + 1 > S.
Texel to point: a, b = (u - 1, v - 1) / (S - 4) for A, (S - 1 - u, S - 1 - v) / (S - 4) for B; negatives to 0; a pair with a + b > 1 divided
by a + b; w0 = (1 - a) - b; P = (w0 v0 + a v1) + b v2.  Normal: (v1 - v0) x (v2 - v0) over sqrt((n0 n0 + n1 n1) + n2 n2), 0 if that is 0.
Colour: the observation weight of every frame at (P, normal) (SDFColorization::computeObservation, as k_recolor), the top-K, and the
weighted mean of the bilinear colours, summed in frame order (K = 0 or at most K observations) or ascending (weight, frame); without an
observation trunc(clamp(((w0 c0 + a c1) + b c2) + 1/2, 0, 255)) of the vertex colours.
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32
CHUNK = 1 << 16                # texels per vectorised block


def layout(F, S):
    ncells = (int(F) + 1) // 2
    cols = math.isqrt(ncells)
    if cols * cols < ncells:
        cols += 1
    rows = -(-ncells // cols)
    return dict(S=int(S), cols=cols, rows=rows, W=cols * S, H=rows * S)


def uv_corners(S, face_b):
    """The UV corners (u, v) of v0, v1, v2 in local texel units, float32 [3, 2]."""
    if face_b:
        return np.array([[S - 1, S - 1], [3, S - 1], [S - 1, 3]], f32)
    return np.array([[1, 1], [S - 3, 1], [1, S - 3]], f32)


def owns(S, face_b, i, j):
    """Whether local texel (i, j) belongs to face B (face_b) or A."""
    i, j = np.asarray(i), np.asarray(j)
    return (i + j + 1 > S) if face_b else (i + j + 1 < S)


def owned_texels(F, S):
    """The owned texels in the kernel's enumeration order (cell-major, row-major inside a cell): face, i, j, and the atlas column x
    and row y, int64 arrays."""
    L = layout(F, S)
    i = np.tile(np.arange(S), S)
    j = np.repeat(np.arange(S), S)
    faces, ii, jj = [], [], []
    for face_b in (False, True):
        m = owns(S, face_b, i, j)
        ncell = (F + 1) // 2 if not face_b else F // 2
        c = np.arange(ncell)
        faces.append((2 * c[:, None] + int(face_b)) + 0 * i[None, m])
        ii.append(np.broadcast_to(i[m], (ncell, int(m.sum()))))
        jj.append(np.broadcast_to(j[m], (ncell, int(m.sum()))))
    face = np.concatenate([f.ravel() for f in faces])
    i = np.concatenate([a.ravel() for a in ii])
    j = np.concatenate([a.ravel() for a in jj])
    c = face // 2
    order = np.argsort(c * S * S + j * S + i, kind="stable")
    face, i, j, c = face[order], i[order], j[order], c[order]
    x = (c % L["cols"]) * S + i
    y = (c // L["cols"]) * S + j
    return face.astype(np.int64), i.astype(np.int64), j.astype(np.int64), x.astype(np.int64), y.astype(np.int64)


def bary(S, face_b, u, v):
    """The clamped (a, b) of local positions (u, v) (float32 arrays) of faces A / B (face_b: bool array)."""
    u, v = np.asarray(u, f32), np.asarray(v, f32)
    L = f32(S - 4)
    e = f32(S - 1)
    a = np.where(face_b, (e - u) / L, (u - f32(1)) / L).astype(f32)
    b = np.where(face_b, (e - v) / L, (v - f32(1)) / L).astype(f32)
    a = np.where(a < 0, f32(0), a)
    b = np.where(b < 0, f32(0), b)
    s = (a + b).astype(f32)
    big = s > 1
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.where(big, a / s, a).astype(f32)
        b = np.where(big, b / s, b).astype(f32)
    return a, b


def point(a, b, p0, p1, p2):
    """P = (w0 v0 + a v1) + b v2 with w0 = (1 - a) - b, float32 [m, 3]; also returns w0."""
    w0 = ((f32(1) - a) - b).astype(f32)
    P = ((w0[:, None] * p0 + a[:, None] * p1) + b[:, None] * p2).astype(f32)
    return P, w0


def face_normals(V, Fc):
    p0, p1, p2 = V[Fc[:, 0]], V[Fc[:, 1]], V[Fc[:, 2]]
    e1, e2 = (p1 - p0).astype(f32), (p2 - p0).astype(f32)
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2], e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]],
                 1).astype(f32)
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2]).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where((ln > 0)[:, None], n / ln[:, None], f32(0)).astype(f32)


def texel_points(mesh, S):
    """Per owned texel in kernel order: face, x, y, a, b, w0, P [m, 3], normal [m, 3]."""
    V = np.asarray(mesh["vertices"], f32).reshape(-1, 3)
    Fc = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    face, i, j, x, y = owned_texels(len(Fc), S)
    fb = (face & 1).astype(bool)
    a, b = bary(S, fb, i.astype(f32) + f32(0.5), j.astype(f32) + f32(0.5))
    P, w0 = point(a, b, V[Fc[face, 0]], V[Fc[face, 1]], V[Fc[face, 2]])
    return dict(face=face, x=x, y=y, a=a, b=b, w0=w0, P=P, N=face_normals(V, Fc)[face])


def uv(F, S):
    """Per-corner OBJ UVs, float32 [F, 3, 2]."""
    L = layout(F, S)
    f = np.arange(F)
    c = f // 2
    x0 = ((c % L["cols"]) * S).astype(f32)
    y0 = ((c // L["cols"]) * S).astype(f32)
    out = np.empty((F, 3, 2), f32)
    for fb in (0, 1):
        m = (f & 1) == fb
        cu = uv_corners(S, bool(fb))
        for k in range(3):
            out[m, k, 0] = (x0[m] + cu[k, 0]) / f32(L["W"])
            out[m, k, 1] = f32(1) - (y0[m] + cu[k, 1]) / f32(L["H"])
    return out


def probe(P, rt, cam, depth):
    """obs_probe: camera point q [m, 3], sub-pixel (pu, pv), depth d under the rounded pixel and ok."""
    R, t = rt[:9].reshape(3, 3).astype(f32), rt[9:].astype(f32)
    q = [(((R[k, 0] * P[:, 0]) + (R[k, 1] * P[:, 1])) + (R[k, 2] * P[:, 2])) + t[k] for k in range(3)]
    with np.errstate(all="ignore"):
        x, y = q[0] / q[2], q[1] / q[2]
        d = cam["d"]
        if np.any(d != 0):
            two, one = f32(2), f32(1)
            r2 = x * x + y * y
            r4 = r2 * r2
            r6 = r4 * r2
            dc = ((one + d[0] * r2) + d[1] * r4) + d[2] * r6
            xn = (x * dc + ((two * d[3]) * x) * y) + d[4] * (r2 + (two * x) * x)
            yn = (y * dc + ((two * d[4]) * xn) * y) + d[3] * (r2 + (two * y) * y)
            x, y = xn, yn
        pu, pv = cam["fx"] * x + cam["cx"], cam["fy"] * y + cam["cy"]
        pu5, pv5 = pu + f32(0.5), pv + f32(0.5)
        lim = f32(2147483000.0)
        ok = (pu5 > -lim) & (pu5 < lim) & (pv5 > -lim) & (pv5 < lim)
        iu = np.where(ok, np.trunc(np.where(ok, pu5, 0)), -1).astype(np.int64)
        iv = np.where(ok, np.trunc(np.where(ok, pv5, 0)), -1).astype(np.int64)
    H, W = depth.shape
    ok &= (iu >= 0) & (iu < W) & (iv >= 0) & (iv < H)
    dd = np.where(ok, depth[np.clip(iv, 0, H - 1), np.clip(iu, 0, W - 1)], f32(0)).astype(f32)
    return np.stack(q, 1).astype(f32), pu.astype(f32), pv.astype(f32), dd, ok


def weight(q, d, ok, N, rt, occlusion):
    """obs_finish: the observation weight, 0 for no observation."""
    R = rt[:9].reshape(3, 3).astype(f32)
    occ = f32(occlusion)
    with np.errstate(all="ignore"):
        valid = ok.copy()
        if occ > 0:
            valid &= (d > 0) & (np.abs(d - q[:, 2]) <= occ)
        valid &= ~(d <= 0)
        nc = np.stack([((R[k, 0] * N[:, 0]) + (R[k, 1] * N[:, 1])) + (R[k, 2] * N[:, 2]) for k in range(3)], 1).astype(f32)
        qn2 = ((q[:, 0] * q[:, 0]) + (q[:, 1] * q[:, 1])) + (q[:, 2] * q[:, 2])
        ql = np.sqrt(qn2)
        v = np.where((qn2 > 0)[:, None], q / ql[:, None], q).astype(f32)
        dt = ((v[:, 0] * nc[:, 0]) + (v[:, 1] * nc[:, 1])) + (v[:, 2] * nc[:, 2])
        w = (f32(1) - np.abs(dt)).astype(f32)
        w = np.where(f32(1) < w, f32(1), w)
        w = np.where(w < f32(0), f32(0), w)
        div = (f32(1) + f32(2) * w).astype(f32)
        rk = (f32(1) / ((div * div) * div)).astype(f32)
        w = np.where(rk < f32(0.001), f32(0.001), rk).astype(f32)
        w = np.where(np.all(nc == 0, 1), f32(0), w)
        return np.where(valid, w, f32(0)).astype(f32)


def interp_u8(img, x, y, ch):
    """interpolate<unsigned char>: bilinear on a B, G, R image, out-of-image taps dropped; float32, truncated."""
    H, W = img.shape[:2]
    fx0, fy0 = np.floor(x).astype(f32), np.floor(y).astype(f32)
    x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
    x1, y1 = x0 + 1, y0 + 1
    x1w, y1w = (x - fx0).astype(f32), (y - fy0).astype(f32)
    x0w, y0w = (f32(1) - x1w).astype(f32), (f32(1) - y1w).astype(f32)
    x0w = np.where((x0 < 0) | (x0 >= W), f32(0), x0w); x1w = np.where((x1 < 0) | (x1 >= W), f32(0), x1w)
    y0w = np.where((y0 < 0) | (y0 >= H), f32(0), y0w); y1w = np.where((y1 < 0) | (y1 >= H), f32(0), y1w)
    w00, w10, w01, w11 = (x0w * y0w).astype(f32), (x1w * y0w).astype(f32), (x0w * y1w).astype(f32), (x1w * y1w).astype(f32)
    sw = (((w00 + w10) + w01) + w11).astype(f32)
    cx0, cx1, cy0, cy1 = np.clip(x0, 0, W - 1), np.clip(x1, 0, W - 1), np.clip(y0, 0, H - 1), np.clip(y1, 0, H - 1)
    acc = np.zeros_like(sw)
    for wgt, yy, xx in ((w00, cy0, cx0), (w01, cy1, cx0), (w10, cy0, cx1), (w11, cy1, cx1)):
        acc = np.where(wgt > 0, (acc + img[yy, xx, ch].astype(f32) * wgt).astype(f32), acc)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(sw > 0, np.trunc(acc / sw), 0).astype(np.uint8)


def _colours(tp, depth, bgr, rt, cam, occlusion, K, vcol, faces):
    """Colours uint8 [m, 3] (R, G, B) and per-texel observation counts for the texels tp (a slice of texel_points)."""
    P, N = tp["P"], tp["N"]
    m, F = len(P), len(rt)
    Wt = np.zeros((m, F), f32)
    PU = np.zeros((m, F), f32)
    PV = np.zeros((m, F), f32)
    for f in range(F):
        q, pu, pv, d, ok = probe(P, rt[f], cam, depth[f])
        Wt[:, f] = weight(q, d, ok, N, rt[f], occlusion)
        PU[:, f], PV[:, f] = pu, pv
    obs = Wt > 0
    n_obs = obs.sum(1)
    fidx = np.broadcast_to(np.arange(F), (m, F))
    if K == 0:
        order = np.argsort(np.where(obs, fidx, F + fidx), axis=1, kind="stable")          # observed frames in frame order first
        n_sel = n_obs
        sel = order
    else:
        key = (Wt.view(np.uint32).astype(np.uint64) << np.uint64(32)) | (fidx + 1).astype(np.uint64)
        by_key = np.argsort(key, axis=1, kind="stable")                                       # ascending (weight, frame)
        by_frame = np.argsort(np.where(obs, fidx, F + fidx), axis=1, kind="stable")
        filt = n_obs > K
        n_sel = np.minimum(n_obs, K)
        # the filter ran: the last K of the ascending keys; otherwise the observed frames in frame order
        start = np.where(filt, F - K, 0)
        cols = start[:, None] + np.arange(max(K, 1))[None, :]
        sel = np.where(filt[:, None], np.take_along_axis(by_key, np.clip(cols, 0, F - 1), 1),
                       np.take_along_axis(by_frame, np.clip(np.arange(max(K, 1))[None, :], 0, F - 1).repeat(m, 0), 1))
    c = np.zeros((m, 3), f32)
    wsum = np.zeros(m, f32)
    scale = f32(1) / f32(255)
    rows = np.arange(m)
    for p in range(int(n_sel.max()) if m else 0):
        act = p < n_sel
        f = sel[:, p]
        w = Wt[rows, f]
        ws = (w * scale).astype(f32)
        for k, ch in enumerate((2, 1, 0)):
            col = np.zeros(m, np.uint8)
            r = np.nonzero(act)[0]
            for fr in np.unique(f[r]):
                rr = r[f[r] == fr]
                col[rr] = interp_u8(bgr[fr], PU[rr, fr], PV[rr, fr], ch)
            c[:, k] = np.where(act, (c[:, k] + col.astype(f32) * ws).astype(f32), c[:, k])
        wsum = np.where(act, (wsum + w).astype(f32), wsum)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (f32(255) / wsum).astype(f32)
        c = np.where((wsum > 0)[:, None], (c * s[:, None]).astype(f32), c)
    out = np.trunc(c).astype(np.uint8)
    # fallback: the barycentric blend of the vertex colours
    none = n_obs == 0
    if none.any():
        fv = faces[tp["face"][none]]
        w0, a, b = tp["w0"][none], tp["a"][none], tp["b"][none]
        for k in range(3):
            c0, c1, c2 = (vcol[fv[:, q], k].astype(f32) for q in range(3))
            x = (((w0 * c0 + a * c1) + b * c2) + f32(0.5)).astype(f32)
            x = np.where(x < 0, f32(0), np.where(x > 255, f32(255), x))
            out[none, k] = np.trunc(x).astype(np.uint8)
    return out, n_obs


def bake(mesh, depth, bgr, rt, cam, S=12, occlusion=0.02, K=5):
    """The texture of mesh (vertices, colors, faces) from frames depth [F, H, W], bgr [F, H, W, 3], poses rt [F, 12] and camera cam
    (render_ref.camera).  Returns dict(image uint8 [H, W, 3], uv float32 [F, 3, 2], info: the counts of I3DTextureInfo except the
    culling's visited count)."""
    V = np.asarray(mesh["vertices"], f32).reshape(-1, 3)
    faces = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    vcol = np.asarray(mesh["colors"], np.uint8).reshape(-1, 3)
    Fn = len(faces)
    L = layout(Fn, S)
    tp = texel_points(mesh, S)
    depth = np.asarray(depth, f32)
    bgr = np.asarray(bgr, np.uint8)
    rt = np.asarray(rt, f32)
    img = np.zeros((L["H"], L["W"], 3), np.uint8)
    n_obs = np.zeros(len(tp["face"]), np.int64)
    for s0 in range(0, len(tp["face"]), CHUNK):
        sl = {k: v[s0:s0 + CHUNK] for k, v in tp.items()}
        col, n = _colours(sl, depth, bgr, rt, cam, occlusion, K, vcol, faces)
        img[sl["y"], sl["x"]] = col
        n_obs[s0:s0 + CHUNK] = n
    owned = len(tp["face"])
    info = dict(atlas_width=L["W"], atlas_height=L["H"], num_faces=Fn, num_texels_owned=owned, num_texels_observed=int((n_obs > 0).sum()),
                num_texels_fallback=int((n_obs == 0).sum()), num_observations=int(n_obs.sum()),
                num_observations_kept=int(n_obs.sum() if K == 0 else np.minimum(n_obs, K).sum()), num_texel_frames_total=owned * len(rt))
    return dict(image=img, uv=uv(Fn, S), info=info)


INFO_COUNTS = ("atlas_width", "atlas_height", "num_faces", "num_texels_owned", "num_texels_observed", "num_texels_fallback", "num_observations",
               "num_observations_kept", "num_texel_frames_total")
