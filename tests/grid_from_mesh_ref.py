"""numpy restatement of the voxel grid from a triangle mesh (i3d_grid_from_mesh, DESIGN.md §6v): the welding, the angle-weighted
pseudonormals, the nearest face and its feature, the sign and the rim rule, and the canonical order.  Shares no code with the kernels; the
nearest face is distance_ref's query, the closest point on it is distance_ref's arithmetic restated once more to return its feature, and
every float64 operation below is one IEEE operation in the order i3d_grid_from_mesh.cuh states, so the grid, the faces and the features
are byte-equal to the device's.

The candidates differ from the device's bricks: every lattice point whose nearest face centroid lies within b + the largest
circumradius (+ a slack) is queried.  The candidates never change a result, only which voxels are looked at."""
import numpy as np
from scipy.spatial import cKDTree

import distance_ref as dr

f32, f64 = np.float32, np.float64
RIM_COS = 0.5           # I3D_GRID_FROM_MESH_RIM_COS


def _dot(x, y):
    return (x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1]) + x[..., 2] * y[..., 2]


def _cross(u, w):
    return np.stack([u[..., 1] * w[..., 2] - u[..., 2] * w[..., 1], u[..., 2] * w[..., 0] - u[..., 0] * w[..., 2],
                     u[..., 0] * w[..., 1] - u[..., 1] * w[..., 0]], -1)


# the feature of a closest point (I3D_FEATURE_*): vertex a, b, c, edge ab, ac, bc, interior; the segments ab, bc, ca as (vertex at t = 0,
# vertex at t = 1, edge)
VERTEX_A, VERTEX_B, VERTEX_C, EDGE_AB, EDGE_AC, EDGE_BC, INTERIOR = range(7)
_SEGMENTS = ((VERTEX_A, VERTEX_B, EDGE_AB), (VERTEX_B, VERTEX_C, EDGE_BC), (VERTEX_C, VERTEX_A, EDGE_AC))


def _seg(p, s0, s1):
    """float32 (d^2, p - q, t) from points p to segments s0 s1, in distance_ref._seg_d2's operations"""
    e = s1 - s0
    sp = p - s0
    ll = dr._dot(e, e)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(ll > 0, dr._dot(sp, e) / np.where(ll > 0, ll, f32(1)), f32(0)).astype(f32)
    t = np.clip(t, f32(0), f32(1))
    d = p - (s0 + t[..., None] * e)
    return dr._dot(d, d), d, t


def point_tri_feature(p, a, b, c):
    """float32 (d^2, feature int8, p - q [N, 3]) from points p [N, 3] to triangles (a, b, c) [N, 3]: the closest point of
    distance_ref.point_tri_d2 (the same operations, so d^2 is byte-equal to it) with the feature it lies on: the procedure's region; for
    the edge fallback the segment of the minimum (ties to ab, then bc, then ca), its end vertex at t = 0 or 1; for a sliver the
    procedure's when its d^2 <= the edges', else the segment's."""
    p, a, b, c = (np.asarray(x, f32) for x in (p, a, b, c))
    ab, ac, ap, bp, cp, bc = b - a, c - a, p - a, p - b, p - c, c - b
    n = np.stack([ab[..., 1] * ac[..., 2] - ab[..., 2] * ac[..., 1], ab[..., 2] * ac[..., 0] - ab[..., 0] * ac[..., 2],
                  ab[..., 0] * ac[..., 1] - ab[..., 1] * ac[..., 0]], -1)
    dot = dr._dot
    d1, d2, d3, d4, d5, d6 = dot(ab, ap), dot(ac, ap), dot(ab, bp), dot(ac, bp), dot(ab, cp), dot(ac, cp)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e43, e56 = d4 - d3, d5 - d6
    conds = [(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
             (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0)]
    region = np.select(conds, [VERTEX_A, VERTEX_B, EDGE_AB, VERTEX_C, EDGE_AC, EDGE_BC], INTERIOR)
    one = np.ones_like(d1)
    num = np.select([region == EDGE_AB, region == EDGE_AC, region == EDGE_BC], [d1, d2, e43], f32(0))
    den = np.select([region == EDGE_AB, region == EDGE_AC, region == EDGE_BC, region == INTERIOR], [d1 - d3, d2 - d6, e43 + e56, (va + vb) + vc], one)
    nn = dot(n, n)
    edges = ~(nn > 0) | ~(den > 0)
    sliver = ~(nn > (dr.SLIVER * dot(ab, ab)) * dot(ac, ac))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        s = (num / den).astype(f32)
        r = (f32(1) / den).astype(f32)
        vi, wi = vb * r, vc * r
    edges |= (region == INTERIOR) & ~((vi >= 0) & (wi >= 0) & (vi + wi <= 1))
    q = np.select([(region == k)[..., None] for k in range(6)],
                  [a, b, c, a + s[..., None] * ab, a + s[..., None] * ac, b + s[..., None] * bc],
                  (a + ab * vi[..., None]) + ac * wi[..., None])
    dv = (p - q).astype(f32)
    out = dot(dv, dv)
    fe = region.astype(np.int8)
    e = edges | sliver
    if e.any():
        pe, ae, be, ce = p[e], a[e], b[e], c[e]
        segs = [_seg(pe, ae, be), _seg(pe, be, ce), _seg(pe, ce, ae)]
        s0, s1, s2 = (sg[0] for sg in segs)
        de = np.minimum(np.minimum(s0, s1), s2)
        w = np.where((s0 <= s1) & (s0 <= s2), 0, np.where(s1 <= s2, 1, 2))
        sf = np.select([w == k for k in range(3)], [np.where(segs[k][2] == 0, v0, np.where(segs[k][2] == 1, v1, ed)) for k, (v0, v1, ed) in
                                                     enumerate(_SEGMENTS)])
        sd = np.select([(w == k)[:, None] for k in range(3)], [segs[k][1] for k in range(3)])
        proc = ~edges[e] & (out[e] <= de)
        fe[e] = np.where(proc, fe[e], sf)
        dv[e] = np.where(proc[:, None], dv[e], sd)
        out[e] = np.where(edges[e], de, np.minimum(out[e], de))
    return out.astype(f32), fe, dv


def weld(vertices):
    """per vertex the lowest index at its exact float position (-0 as +0)"""
    v = np.asarray(vertices, f32)
    bits = np.where(v == 0, f32(0), v).view(np.uint32)
    _, inv = np.unique(bits, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    rep = np.full(inv.max() + 1, len(v), np.int64)
    np.minimum.at(rep, inv, np.arange(len(v)))
    return rep[inv]


def topology(mesh):
    """unit face normals fn [F, 3], per corner 3 f + k the vertex pseudonormal vn and per edge slot 3 f + k (corners k, k + 1) the edge
    pseudonormal en [3F, 3] and boundary flag eb, per vertex the welded boundary flag vb and the weld representative"""
    v = np.asarray(mesh["vertices"], f32)
    f = np.asarray(mesh["faces"], np.int64)
    F = len(f)
    rep = weld(v)
    V64 = v.astype(f64)
    n = _cross(V64[f[:, 1]] - V64[f[:, 0]], V64[f[:, 2]] - V64[f[:, 0]])
    nn = _dot(n, n)
    deg = ~(nn > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        fn = np.where(deg[:, None], 0.0, n / np.sqrt(nn)[:, None])
    inc_f = np.repeat(np.arange(F), 3)
    inc_k = np.tile(np.arange(3), F)
    corner = f[inc_f, inc_k]
    nxt, prv = f[inc_f, (inc_k + 1) % 3], f[inc_f, (inc_k + 2) % 3]
    ok = ~deg[inc_f]
    # vertex pseudonormals: sum of angle * unit normal over the incidences in ascending face id (np.add.at runs in index order)
    u, w = V64[nxt] - V64[corner], V64[prv] - V64[corner]
    x = _cross(u, w)
    ang = np.arctan2(np.sqrt(_dot(x, x)), _dot(u, w))
    wv = rep[corner]
    acc = np.zeros((len(v), 3))
    np.add.at(acc, wv[ok], ang[ok][:, None] * fn[inc_f[ok]])
    vn = acc[wv]
    # edge pseudonormals and the boundary: welded pairs
    ra, rb = rep[corner], rep[nxt]
    pair = np.stack([np.minimum(ra, rb), np.maximum(ra, rb)], 1)
    _, eg = np.unique(pair, axis=0, return_inverse=True)
    eg = eg.reshape(-1)
    eacc = np.zeros((eg.max() + 1, 3))
    np.add.at(eacc, eg[ok], fn[inc_f[ok]])
    used = np.zeros(eg.max() + 1, np.int64)
    np.add.at(used, eg[ok], 1)
    en = eacc[eg]
    eb = used[eg] == 1
    vb = np.zeros(len(v), bool)
    vb[pair[eb].reshape(-1)] = True
    return dict(fn=fn, vn=vn, en=en, eb=eb, vb=vb, rep=rep, num_welded=len(np.unique(rep)), num_boundary_edges=int((used == 1).sum()))


def order_key(xyz):
    """fuse_order_key: (bz, by, bx, lz, ly, lx) of c + 2^20, unsigned (bz takes the top bit)"""
    u = (np.asarray(xyz, np.int64) + (1 << 20)).astype(np.uint64)
    s = lambda k: np.uint64(k)  # noqa: E731
    return (((u[:, 2] >> s(3)) << s(46)) | ((u[:, 1] >> s(3)) << s(28)) | ((u[:, 0] >> s(3)) << s(10)) | ((u[:, 2] & s(7)) << s(6))
            | ((u[:, 1] & s(7)) << s(3)) | (u[:, 0] & s(7)))


def candidates(mesh, voxel_size, band, slab=1 << 22):
    """the lattice points within b + the largest circumradius (+ slack) of a face centroid, int32 [N, 3]"""
    v = np.asarray(mesh["vertices"], f32).astype(f64)
    f = np.asarray(mesh["faces"], np.int64)
    vs, b = float(f32(voxel_size)), float(f32(band) * f32(voxel_size))
    cen = (v[f[:, 0]] + v[f[:, 1]] + v[f[:, 2]]) / 3.0
    rad = max(np.linalg.norm(v[f[:, k]] - cen, axis=1).max() for k in range(3))
    reach = b + rad + 1e-6 * (1.0 + np.abs(v).max()) + 1e-3 * vs
    tree = cKDTree(cen)
    lo = np.floor((v.min(0) - b) / vs).astype(np.int64) - 1
    hi = np.ceil((v.max(0) + b) / vs).astype(np.int64) + 1
    xs, ys, zs = (np.arange(lo[k], hi[k] + 1) for k in range(3))
    out = []
    zstep = max(1, slab // (len(xs) * len(ys)))
    for z0 in range(0, len(zs), zstep):
        Z, Y, X = np.meshgrid(zs[z0:z0 + zstep], ys, xs, indexing="ij")
        c = np.stack([X, Y, Z], -1).reshape(-1, 3)
        d, _ = tree.query(c * vs, distance_upper_bound=reach)
        out.append(c[np.isfinite(d)])
    return np.concatenate(out).astype(np.int32)


def grid_from_mesh(mesh, voxel_size, band=3.0, topo=None):
    """the grid i3d_grid_from_mesh installs: xyz int32 [n, 3] in canonical order, sdf float64 [n], face int32 [n], feature int8 [n],
    and the drop counts of the voxels within the band"""
    v = np.asarray(mesh["vertices"], f32)
    f = np.asarray(mesh["faces"], np.int64)
    vs = f32(voxel_size)
    b = f32(band) * vs
    t = topology(mesh) if topo is None else topo
    c = candidates(mesh, voxel_size, band)
    P = c.astype(f32) * vs
    d2, face = dr.nearest(P, mesh, b)
    m = face >= 0
    c, P, d2, face = c[m], P[m], d2[m], face[m].astype(np.int64)
    d2r, feat, dv = point_tri_feature(P, v[f[face, 0]], v[f[face, 1]], v[f[face, 2]])
    assert d2r.tobytes() == d2.tobytes()
    slot = np.select([feat == EDGE_AB, feat == EDGE_BC], [0, 1], 2)
    vert = np.minimum(feat, 2)
    N = np.select([(feat == INTERIOR)[:, None], (feat <= VERTEX_C)[:, None]], [t["fn"][face], t["vn"][3 * face + vert]], t["en"][3 * face + slot])
    boundary = np.select([feat == INTERIOR, feat <= VERTEX_C], [False, t["vb"][t["rep"][f[face, vert]]]], t["eb"][3 * face + slot])
    d = dv.astype(f64)
    dot, dd, nn = _dot(d, N), _dot(d, d), _dot(N, N)
    zero = d2 == 0
    zero_normal = ~zero & (nn == 0)
    zero_dot = ~zero & ~zero_normal & (dot == 0)
    rim = ~zero & ~zero_normal & ~zero_dot & boundary & (dot * dot < ((RIM_COS * RIM_COS) * dd) * nn)
    keep = ~(zero_normal | zero_dot | rim)
    r = np.sqrt(d2).astype(f64)
    sdf = np.where(zero, 0.0, np.where(dot > 0, r, -r))
    o = np.argsort(order_key(c[keep]), kind="stable")
    return dict(xyz=c[keep][o], sdf=sdf[keep][o], face=face[keep][o].astype(np.int32), feature=feat[keep][o].astype(np.int8),
                num_dropped_rim=int(rim.sum()), num_dropped_zero_normal=int(zero_normal.sum()), num_dropped_zero_dot=int(zero_dot.sum()),
                num_negative=int((sdf[keep] < 0).sum()), num_welded=t["num_welded"], num_boundary_edges=t["num_boundary_edges"])


def face_normal_signs(mesh, out, voxel_size):
    """the sign the nearest face's own normal gives each voxel of `out`, sign(dot(p - q, n)): the rule the pseudonormals replace"""
    v = np.asarray(mesh["vertices"], f32)
    f = np.asarray(mesh["faces"], np.int64)[out["face"].astype(np.int64)]
    P = out["xyz"].astype(f32) * f32(voxel_size)
    _, _, dv = point_tri_feature(P, v[f[:, 0]], v[f[:, 1]], v[f[:, 2]])
    V64 = v.astype(f64)
    n = _cross(V64[f[:, 1]] - V64[f[:, 0]], V64[f[:, 2]] - V64[f[:, 0]])
    return np.sign(_dot(dv.astype(f64), n))


# ---- test meshes ---------------------------------------------------------------------------------------------------------------------
_CUBE_V = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]], f64)
_CUBE_F = np.array([[0, 2, 1], [0, 3, 2], [4, 5, 6], [4, 6, 7], [0, 1, 5], [0, 5, 4], [1, 2, 6], [1, 6, 5], [2, 3, 7], [2, 7, 6],
                    [3, 0, 4], [3, 4, 7]], np.int64)


def box_mesh(lo, hi, R=np.eye(3), t=np.zeros(3)):
    """a closed box [lo, hi] (outward winding), rotated by R and moved by t, float32"""
    lo, hi = np.asarray(lo, f64), np.asarray(hi, f64)
    v = (lo + _CUBE_V * (hi - lo)) @ np.asarray(R, f64).T + t
    return dict(vertices=v.astype(f32), faces=_CUBE_F.astype(np.int32), colors=np.zeros((8, 3), np.uint8))


def split_vertices(mesh):
    """the same mesh with three vertices of its own per face, as STL and many OBJ exports store it"""
    v = np.asarray(mesh["vertices"], f32)
    f = np.asarray(mesh["faces"], np.int64)
    return dict(vertices=v[f.reshape(-1)].copy(), faces=np.arange(3 * len(f), dtype=np.int32).reshape(-1, 3), colors=np.zeros((3 * len(f), 3), np.uint8))


def box_sdf(p, lo, hi, R=np.eye(3), t=np.zeros(3)):
    """float64 signed distance to the box of box_mesh"""
    q = (np.asarray(p, f64) - t) @ np.asarray(R, f64)
    c, h = (np.asarray(lo, f64) + np.asarray(hi, f64)) / 2, (np.asarray(hi, f64) - np.asarray(lo, f64)) / 2
    d = np.abs(q - c) - h
    return np.linalg.norm(np.maximum(d, 0.0), axis=-1) + np.minimum(d.max(-1), 0.0)


def _prism(pts, caps, h, t):
    """the polygon pts [n, 2] (counter-clockwise; bottom cap triangles `caps`, normal -z) extruded over [0, h] in z and moved by t: a closed
    mesh and its float64 signed distance (the polygon's 2-D signed distance extruded)"""
    n = len(pts)
    v = np.concatenate([np.c_[pts, np.zeros(n)], np.c_[pts, np.full(n, h)]]) + t
    faces = [list(f) for f in caps] + [[n + a, n + c, n + b] for a, b, c in caps]
    for i in range(n):
        j = (i + 1) % n
        faces += [[i, j, n + j], [i, n + j, n + i]]
    mesh = dict(vertices=v.astype(f32), faces=np.array(faces, np.int32), colors=np.zeros((2 * n, 3), np.uint8))

    def sdf(p):
        q = np.asarray(p, f64) - t
        a, b = pts, np.roll(pts, -1, axis=0)
        e = b - a
        xy = q[:, None, :2] - a[None]
        tt = np.clip((xy * e[None]).sum(-1) / (e * e).sum(-1)[None], 0.0, 1.0)
        d2d = np.linalg.norm(xy - tt[..., None] * e[None], axis=-1).min(1)
        # even-odd crossings of a ray along +x
        y0, y1 = a[None, :, 1], b[None, :, 1]
        cross = ((y0 > q[:, None, 1]) != (y1 > q[:, None, 1])) & (q[:, None, 0] < a[None, :, 0] + (q[:, None, 1] - y0) * (b[None, :, 0] - a[None, :, 0]) / np.where(y1 != y0, y1 - y0, 1.0))
        inside = cross.sum(1) % 2 == 1
        w = np.stack([np.where(inside, -d2d, d2d), np.abs(q[:, 2] - h / 2) - h / 2], 1)
        return np.minimum(w.max(1), 0.0) + np.linalg.norm(np.maximum(w, 0.0), axis=1)
    return mesh, sdf


def l_prism(s, t):
    """an L-shaped prism: the union of [0, 2s] x [0, s] x [0, s] and [0, s] x [0, 2s] x [0, s], moved by t; a closed mesh with a
    concave edge along x = y = s and concave vertices at its ends"""
    pts = np.array([[0, 0], [2, 0], [2, 1], [1, 1], [1, 2], [0, 2]], f64) * s
    return _prism(pts, [[0, 2, 1], [0, 3, 2], [0, 5, 3], [3, 5, 4]], s, t)


def wedge(length, apex_deg, h, t):
    """a knife-edged triangular prism: an isosceles triangle with an apex angle of apex_deg (a convex edge sharper than 90 degrees, where
    the nearest face's own normal gives the wrong sign), extruded over [0, h]"""
    half = np.radians(apex_deg) / 2
    pts = np.array([[0, 0], [length, -length * np.tan(half)], [length, length * np.tan(half)]], f64)
    return _prism(pts, [[0, 2, 1]], h, t)


def square_patch(lo, hi, z, n=2):
    """an open n x n grid of squares (two triangles each) over [lo, hi]^2 at height z, normal +z"""
    g = np.linspace(lo, hi, n + 1)
    X, Y = np.meshgrid(g, g, indexing="xy")
    v = np.c_[X.reshape(-1), Y.reshape(-1), np.full(X.size, z)]
    faces = []
    for j in range(n):
        for i in range(n):
            a, b, c, d = j * (n + 1) + i, j * (n + 1) + i + 1, (j + 1) * (n + 1) + i + 1, (j + 1) * (n + 1) + i
            faces += [[a, b, c], [a, c, d]]
    return dict(vertices=v.astype(f32), faces=np.array(faces, np.int32), colors=np.zeros((len(v), 3), np.uint8))
