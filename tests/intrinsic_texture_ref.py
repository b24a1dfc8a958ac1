"""numpy float32 restatement of the texture decomposition and the relit raster (DESIGN.md §6x; i3d_texture.cuh k_tex_decompose,
i3d_raster.cuh rast_relit), built on texture_ref (texel points and normals, the bake's observation weight), vis_ref (the SH blend and the
shading dot product) and raster_ref (the hits and their statistics).  Every float operation is one numpy float32 operation in the order
the kernels state, so the atlases, planes and counts are byte-equal to the device's.

Lighting: a function of the points P float32 [m, 3] giving the float SH [m, 9]: global_sh(sh) (the same nine floats everywhere) or
estimate_sh(sub_index, sub_sh, subvolume_size) (the one subvolume's SH when there is one, else the blend at P, rounded to float).
Decomposition per owned texel: s = sh . basis(n) at the bake's P and face normal n; lit iff n != 0 and s > min_shading; A_k = (c_k / 255)
/ s of the baked colour, 0 when unlit; shading = s where n != 0, else 0; unowned texels 0.
Relit colour of a hit: the texture source's clamped (a, b) and lookup position, A = interp_f32 of the albedo atlas there, s' at the
hit face's normal and at P = (w0 p0 + a p1) + b p2 of the clamped (a, b); per channel trunc(clamp((A s') 255 + 1/2, 0, 255)); 0 for a
zero normal.
"""
from __future__ import annotations

import numpy as np

import raster_ref as ra
import texture_ref as tr
import vis_ref

f32 = np.float32


def global_sh(sh):
    v = np.asarray(sh, f32).reshape(9)
    return lambda P: np.broadcast_to(v, (len(P), 9)).astype(f32)


def blend_at(P, sub_index, sub_sh, subvolume_size):
    """vis_ref.blend_sh's rule at world points P float32 [m, 3] instead of voxel centres: float64 [m, 9]."""
    inv = f32(1) / f32(subvolume_size)
    pos = (np.asarray(P, f32) * inv - f32(0.5)).astype(f32)
    fl = np.floor(pos)
    v0 = fl.astype(np.int64)
    wg = (pos - fl).astype(f32)
    look = vis_ref._Lookup(np.asarray(sub_index, np.int64))
    sub_sh = np.asarray(sub_sh, np.float64)
    n = len(pos)
    avg = np.zeros((n, 9), np.float64)
    sum_w = np.zeros(n, f32)
    for c in vis_ref.CORNERS:
        wx = np.where(c[0] == 1, wg[:, 0], f32(1) - wg[:, 0])
        wy = np.where(c[1] == 1, wg[:, 1], f32(1) - wg[:, 1])
        wz = np.where(c[2] == 1, wg[:, 2], f32(1) - wg[:, 2])
        w = ((wx * wy) * wz).astype(f32)
        sid = look(v0 + c)
        use = (sid >= 0) & (w != 0)
        prod = w.astype(np.float64)[:, None] * sub_sh[np.maximum(sid, 0)]
        first = (sum_w == 0)[:, None]
        avg = np.where(use[:, None], np.where(first, prod, avg + prod), avg)
        sum_w = np.where(use, sum_w + w, sum_w).astype(f32)
    nz = sum_w != 0
    with np.errstate(divide="ignore"):
        scale = (f32(1) / np.where(nz, sum_w, f32(1))).astype(np.float64)
    return np.where(nz[:, None], avg * scale[:, None], avg)


def estimate_sh(sub_index, sub_sh, subvolume_size):
    sub_sh = np.asarray(sub_sh, np.float64).reshape(-1, 9)
    if len(sub_sh) == 1:
        return lambda P: np.broadcast_to(sub_sh[0].astype(f32), (len(P), 9)).astype(f32)
    return lambda P: blend_at(P, sub_index, sub_sh, subvolume_size).astype(f32)


def sh_dot(N, sh):
    """sh . basis(n): vis_ref.shading at albedo 1 (1 * d is d itself)."""
    return vis_ref.shading(np.asarray(N, f32), np.asarray(sh, f32), np.ones(len(N), f32))


def observed(mesh, depth, rt, cam, S, occlusion=0.02):
    """The bake's per-texel observation flag, bool [H, W]: some frame gives the texel's point and normal a weight > 0."""
    L = tr.layout(len(np.asarray(mesh["faces"]).reshape(-1, 3)), S)
    tp = tr.texel_points(mesh, S)
    out = np.zeros((L["H"], L["W"]), bool)
    rt = np.asarray(rt, f32)
    depth = np.asarray(depth, f32)
    for s0 in range(0, len(tp["face"]), tr.CHUNK):
        P, N = tp["P"][s0:s0 + tr.CHUNK], tp["N"][s0:s0 + tr.CHUNK]
        obs = np.zeros(len(P), bool)
        for f in range(len(rt)):
            q, pu, pv, d, ok = tr.probe(P, rt[f], cam, depth[f])
            obs |= tr.weight(q, d, ok, N, rt[f], occlusion) > 0
        out[tp["y"][s0:s0 + tr.CHUNK], tp["x"][s0:s0 + tr.CHUNK]] = obs
    return out


def decompose(image, mesh, S, lighting, min_shading=0.05, observed_mask=None):
    """The decomposition of the baked atlas image uint8 [H, W, 3] of mesh at S texels per face under lighting (global_sh / estimate_sh).
    observed_mask bool [H, W] (observed(); None: every texel observed).  Returns dict(albedo float32 [H, W, 3], shading float32 [H, W],
    info: the counts and albedo range of I3DIntrinsicTextureInfo)."""
    image = np.asarray(image, np.uint8)
    H, W = image.shape[:2]
    tp = tr.texel_points(mesh, S)
    N, P, x, y = tp["N"], tp["P"], tp["x"], tp["y"]
    nz = ~np.all(N == 0, 1)
    s = np.where(nz, sh_dot(N, lighting(P)), f32(0)).astype(f32)
    lit = nz & (s > f32(min_shading))
    c = image[y, x].astype(f32)
    with np.errstate(all="ignore"):
        A = np.where(lit[:, None], ((c / f32(255)).astype(f32) / s[:, None]).astype(f32), f32(0)).astype(f32)
    albedo = np.zeros((H, W, 3), f32)
    shading = np.zeros((H, W), f32)
    albedo[y, x] = A
    shading[y, x] = s
    obs = np.ones(len(x), bool) if observed_mask is None else observed_mask[y, x]
    info = dict(atlas_width=W, atlas_height=H, num_texels_owned=len(x), num_texels_lit=int(lit.sum()), num_texels_unlit=int((~lit).sum()),
                num_texels_lit_fallback=int((lit & ~obs).sum()),
                albedo_min=[float(A[lit, k].min()) if lit.any() else 0.0 for k in range(3)],
                albedo_max=[float(A[lit, k].max()) if lit.any() else 0.0 for k in range(3)])
    return dict(albedo=albedo, shading=shading, info=info)


INFO_COUNTS = ("atlas_width", "atlas_height", "num_texels_owned", "num_texels_lit", "num_texels_unlit", "num_texels_lit_fallback")


def interp_f32(img, x, y, ch):
    """interp_u8's bilinear lookup on a float32 [H, W, 3] image without the truncation; 0 where no tap has weight."""
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
        return np.where(sw > 0, acc / sw, f32(0)).astype(f32)


def lookup(face, a, b, S, cols):
    """The texture source's clamped (ac, bc) and atlas position (X, Y) of hits (face, a, b)."""
    ac, bc = np.where(a < 0, f32(0), a).astype(f32), np.where(b < 0, f32(0), b).astype(f32)
    s = (ac + bc).astype(f32)
    big = s > 1
    with np.errstate(all="ignore"):
        ac = np.where(big, ac / s, ac).astype(f32)
        bc = np.where(big, bc / s, bc).astype(f32)
    w = ((f32(1) - ac) - bc).astype(f32)
    fb = (face & 1).astype(bool)
    cu = np.where(fb[:, None, None], tr.uv_corners(S, True)[None], tr.uv_corners(S, False)[None])
    u = ((w * cu[:, 0, 0] + ac * cu[:, 1, 0]) + bc * cu[:, 2, 0]).astype(f32)
    v = ((w * cu[:, 0, 1] + ac * cu[:, 1, 1]) + bc * cu[:, 2, 1]).astype(f32)
    cell = face // 2
    X = ((((cell % cols) * S).astype(f32) + u) - f32(0.5)).astype(f32)
    Y = ((((cell // cols) * S).astype(f32) + v) - f32(0.5)).astype(f32)
    return ac, bc, X, Y


def relit_colour(mesh, face, a, b, albedo, S, lighting):
    """The relit colour uint8 [m, 3] of hits (face, a, b) of mesh from the albedo atlas at S texels per face."""
    V = np.asarray(mesh["vertices"], f32).reshape(-1, 3)
    Fc = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    cols = tr.layout(len(Fc), S)["cols"]
    ac, bc, X, Y = lookup(face, a, b, S, cols)
    P, _ = tr.point(ac, bc, V[Fc[face, 0]], V[Fc[face, 1]], V[Fc[face, 2]])
    N = tr.face_normals(V, Fc)[face]
    s = sh_dot(N, lighting(P))
    out = np.zeros((len(face), 3), np.uint8)
    for k in range(3):
        A = interp_f32(albedo, X, Y, k)
        x = (((A * s).astype(f32) * f32(255)).astype(f32) + f32(0.5)).astype(f32)
        out[:, k] = np.trunc(np.clip(x, f32(0), f32(255))).astype(np.uint8)
    out[np.all(N == 0, 1)] = 0
    return out


def rasterize(mesh, rts, cam, W, H, albedo, S, lighting, depth=None, bgr=None, ids=None):
    """raster_ref.rasterize with the relit colour source: the same planes and statistics, the colour planes and colour pairs relit."""
    out = ra.rasterize(mesh, rts, cam, W, H, color=None, depth=depth, ids=ids)
    views = list(ids) if ids is not None else list(range(len(rts)))
    for i, vi in enumerate(views):
        face = out["face"][i].reshape(-1)
        p = np.nonzero(face >= 0)[0]
        bar = out["bary"][i].reshape(-1, 2)
        rgb = out["rgb"][i].reshape(-1, 3)
        rgb[p] = relit_colour(mesh, face[p].astype(np.int64), bar[p, 0], bar[p, 1], albedo, S, lighting)
        if depth is not None and bgr is not None:
            fr = np.asarray(bgr[vi], np.uint8).reshape(-1, 3)
            ec = rgb[p].astype(np.int64) - fr[p][:, ::-1].astype(np.int64)
            st = out["stats"][i]
            st["color_count"] = int(len(p))
            st["color_abs"] = [int(v) for v in np.abs(ec).sum(0)]
            st["color_sq"] = [int(v) for v in (ec * ec).sum(0)]
    return out
