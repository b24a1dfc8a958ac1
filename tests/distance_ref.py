"""numpy float32 restatement of the surface distance (i3d_surface_distance, DESIGN.md §6u): the samples, the closest point on a triangle,
the nearest-face query and the float64 statistics.  Shares no code with the kernels; every float32 operation below is one IEEE operation
in the order i3d_distance.cuh states, so (d^2, face) per sample and per vertex are byte-equal to the device's.

Two queries give the same answer, the lexicographic minimum of (float32 d^2, face id) over every face with d^2 <= max_distance^2:
nearest_brute tests every face; nearest prunes with a k-d tree over the face centroids, an acceleration unlike the device's grid, so
agreement with it is also a check that the grid changes nothing."""
import numpy as np
from scipy.spatial import cKDTree

f32 = np.float32
INF = f32(np.inf)
SLIVER = f32(2.0 ** -20)      # kDistSliver


def _dot(x, y):
    return (x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1]) + x[..., 2] * y[..., 2]


def _seg_d2(p, s0, s1):
    e = s1 - s0
    sp = p - s0
    ll = _dot(e, e)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(ll > 0, _dot(sp, e) / np.where(ll > 0, ll, f32(1)), f32(0)).astype(f32)
    t = np.clip(t, f32(0), f32(1))
    d = p - (s0 + t[..., None] * e)
    return _dot(d, d)


def point_tri_d2(p, a, b, c):
    """float32 d^2 from points p [N, 3] to triangles (a, b, c) [N, 3] each (broadcasting): Ericson's closest point, the edge fallback"""
    p, a, b, c = (np.asarray(x, f32) for x in (p, a, b, c))
    p, a, b, c = np.broadcast_arrays(p, a, b, c)
    ab, ac, ap, bp, cp, bc = b - a, c - a, p - a, p - b, p - c, c - b
    n = np.stack([ab[..., 1] * ac[..., 2] - ab[..., 2] * ac[..., 1], ab[..., 2] * ac[..., 0] - ab[..., 0] * ac[..., 2],
                  ab[..., 0] * ac[..., 1] - ab[..., 1] * ac[..., 0]], -1)
    d1, d2, d3, d4, d5, d6 = _dot(ab, ap), _dot(ac, ap), _dot(ab, bp), _dot(ac, bp), _dot(ab, cp), _dot(ac, cp)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e43, e56 = d4 - d3, d5 - d6
    conds = [(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
             (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0)]
    region = np.select(conds, [0, 1, 3, 2, 4, 5], 6)        # vertex a, vertex b, edge ab, vertex c, edge ac, edge bc, interior
    one = np.ones_like(d1)
    num = np.select([region == 3, region == 4, region == 5], [d1, d2, e43], f32(0))
    den = np.select([region == 3, region == 4, region == 5, region == 6], [d1 - d3, d2 - d6, e43 + e56, (va + vb) + vc], one)
    nn = _dot(n, n)
    edges = ~(nn > 0) | ~(den > 0)
    sliver = ~(nn > (SLIVER * _dot(ab, ab)) * _dot(ac, ac))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        s = (num / den).astype(f32)
        r = (f32(1) / den).astype(f32)
        vi, wi = vb * r, vc * r
    edges |= (region == 6) & ~((vi >= 0) & (wi >= 0) & (vi + wi <= 1))
    q = np.select([(region == k)[..., None] for k in range(6)],
                  [a, b, c, a + s[..., None] * ab, a + s[..., None] * ac, b + s[..., None] * bc],
                  (a + ab * vi[..., None]) + ac * wi[..., None])
    d = p - q
    out = _dot(d, d)
    e = edges | sliver
    if e.any():
        pe, ae, be, ce = p[e], a[e], b[e], c[e]
        de = np.minimum(np.minimum(_seg_d2(pe, ae, be), _seg_d2(pe, be, ce)), _seg_d2(pe, ce, ae))
        out[e] = np.where(edges[e], de, np.minimum(out[e], de))
    return out.astype(f32)


def sample_bary(L):
    """(a, b) float32 [L^2] of the samples of a face in sample order: the up sub-triangles, then the down ones"""
    third, two_thirds = f32(1) / f32(3), f32(2) / f32(3)
    ij = [(i, j, third) for i in range(L) for j in range(L - i)] + [(i, j, two_thirds) for i in range(L - 1) for j in range(L - 1 - i)]
    a = np.array([(f32(i) + o) / f32(L) for i, _, o in ij], f32)
    b = np.array([(f32(j) + o) / f32(L) for _, j, o in ij], f32)
    return a, b


def face_area(v, f):
    """float32 area of every face, in the kernels' order"""
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    n0 = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    n1 = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    n2 = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    return f32(0.5) * np.sqrt((n0 * n0 + n1 * n1) + n2 * n2)


def samples(mesh, L):
    """points float32 [F L^2, 3] in sample order (face-major) and weights float64 [F L^2] = double(area) / L^2"""
    v = np.asarray(mesh["vertices"], f32)
    f = np.asarray(mesh["faces"], np.int64)
    a, b = sample_bary(L)
    w0 = (f32(1) - a) - b
    p0, p1, p2 = v[f[:, 0]][:, None, :], v[f[:, 1]][:, None, :], v[f[:, 2]][:, None, :]
    P = ((w0[None, :, None] * p0 + a[None, :, None] * p1) + b[None, :, None] * p2).reshape(-1, 3)
    w = np.repeat(face_area(v, f).astype(np.float64) / np.float64(L * L), L * L)
    return P.astype(f32), w


def _lexmin(pt, fc, d2, n):
    """per point the (d^2, face) lexicographic minimum over its candidate pairs (pt, fc, d2); (inf, -1) without one"""
    out_d2 = np.full(n, INF, f32)
    out_f = np.full(n, -1, np.int32)
    if len(pt):
        o = np.lexsort((fc, d2, pt))
        pt, fc, d2 = pt[o], fc[o], d2[o]
        first = np.ones(len(pt), bool)
        first[1:] = pt[1:] != pt[:-1]
        out_d2[pt[first]] = d2[first]
        out_f[pt[first]] = fc[first]
    return out_d2, out_f


def nearest_brute(P, mesh, max_distance, chunk=1 << 20):
    """every face against every point"""
    v = np.asarray(mesh["vertices"], f32)
    f = np.asarray(mesh["faces"], np.int64)
    lim = f32(max_distance) * f32(max_distance)
    P = np.asarray(P, f32)
    d2o = np.full(len(P), INF, f32)
    fo = np.full(len(P), -1, np.int32)
    step = max(1, chunk // max(1, len(f)))
    for s in range(0, len(P), step):
        p = P[s:s + step]
        d = point_tri_d2(p[:, None, :], v[f[:, 0]][None], v[f[:, 1]][None], v[f[:, 2]][None])
        d = np.where(d <= lim, d, INF)
        k = np.argmin(d, axis=1)                     # the first minimum: the lowest face id among equal d^2
        dk = d[np.arange(len(p)), k]
        ok = dk <= lim
        d2o[s:s + step] = np.where(ok, dk, INF)
        fo[s:s + step] = np.where(ok, k, -1)
    return d2o, fo


def nearest(P, mesh, max_distance, chunk=1 << 18):
    """the same answer as nearest_brute: the faces whose centroid lies within sqrt(bound) + their circumradius (+ a slack far above
    float rounding) of the point, bound = min(max_distance^2, d^2 to the face of the nearest centroid)"""
    v = np.asarray(mesh["vertices"], f32)
    f = np.asarray(mesh["faces"], np.int64)
    P = np.asarray(P, f32)
    lim = f32(max_distance) * f32(max_distance)
    v64 = v.astype(np.float64)
    cen = (v64[f[:, 0]] + v64[f[:, 1]] + v64[f[:, 2]]) / 3.0
    rad = np.max(np.stack([np.linalg.norm(v64[f[:, k]] - cen, axis=1) for k in range(3)]), axis=0)
    tree = cKDTree(cen)
    slack = 1e-5 * (1.0 + np.abs(v64).max() + np.abs(P).max())
    d2o = np.empty(len(P), f32)
    fo = np.empty(len(P), np.int32)
    for s in range(0, len(P), chunk):
        p = P[s:s + chunk]
        p64 = p.astype(np.float64)
        _, k0 = tree.query(p64)
        ub = point_tri_d2(p, v[f[k0, 0]], v[f[k0, 1]], v[f[k0, 2]])
        bound = np.sqrt(np.minimum(ub, lim).astype(np.float64))
        cand = tree.query_ball_point(p64, bound + rad.max() + slack)
        cnt = np.fromiter((len(c) for c in cand), np.int64, len(cand))
        pt = np.repeat(np.arange(len(p)), cnt)
        fc = np.fromiter((x for c in cand for x in c), np.int64, int(cnt.sum()))
        keep = np.linalg.norm(p64[pt] - cen[fc], axis=1) <= bound[pt] + rad[fc] + slack
        pt, fc = pt[keep], fc[keep]
        d2 = point_tri_d2(p[pt], v[f[fc, 0]], v[f[fc, 1]], v[f[fc, 2]])
        ok = d2 <= lim
        d2o[s:s + chunk], fo[s:s + chunk] = _lexmin(pt[ok], fc[ok].astype(np.int32), d2[ok], len(p))
    return d2o, fo


def side_stats(d2, face, w, thresholds):
    """float64 statistics of one direction from its per-sample (d^2, face) and weights"""
    m = face >= 0
    d = np.sqrt(d2[m].astype(np.float64))
    wm = w[m]
    am = wm.sum()
    out = dict(num_samples=len(d2), num_matched=int(m.sum()), area=float(w.sum()), unmatched_area=float(w[~m].sum()),
               mean=float((wm * d).sum() / am) if am > 0 else 0.0, rms=float(np.sqrt((wm * d2[m].astype(np.float64)).sum() / am)) if am > 0 else 0.0,
               max=float(d.max()) if len(d) else 0.0)
    tot = w.sum()
    out["fraction"] = [float(wm[d2[m] <= f32(t) * f32(t)].sum() / tot) if tot > 0 else 0.0 for t in thresholds]
    return out


def distance(mesh_a, mesh_b, L, max_distance, thresholds=(), query=nearest):
    """both directions and the vertex query of mesh_a against mesh_b, as i3d_surface_distance computes them"""
    out = {}
    for name, src, tgt in (("accuracy", mesh_a, mesh_b), ("completeness", mesh_b, mesh_a)):
        P, w = samples(src, L)
        d2, fc = query(P, tgt, max_distance)
        out[name] = side_stats(d2, fc, w, thresholds)
        out[name + "_d2"], out[name + "_face"] = d2, fc
    P, R = out["accuracy"]["fraction"], out["completeness"]["fraction"]
    out["precision"], out["recall"] = P, R
    out["fscore"] = [2 * p * r / (p + r) if p + r > 0 else 0.0 for p, r in zip(P, R)]
    vd2, vf = query(np.asarray(mesh_a["vertices"], f32), mesh_b, max_distance)
    out["vertex_distance"] = np.where(vf >= 0, np.sqrt(vd2), INF).astype(f32)
    out["vertex_face"] = vf
    return out
