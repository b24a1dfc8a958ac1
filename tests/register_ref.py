"""numpy restatement of the reference-mesh registration (i3d_register_reference_mesh, DESIGN.md §6aa): point-to-plane ICP of the resident
mesh's area samples against the reference mesh's faces, in float32 and float64 in the order i3d_register.cuh states.

The samples and the nearest face are distance_ref's, the closest point on that face is grid_from_mesh_ref's (the same operations, with
p - q), and the solve and the pose update are track_ref's.  Every float32 operation is one IEEE operation, every float64 one as well, and
the sums follow the device's order (per 256-sample block a warp shuffle tree and the warps in order, then the blocks in order), so a
system formed at the same float pose is the device's bit for bit; poses after an update agree to the last bits (track_ref's sin / cos).

T maps the reference B onto the resident A (x_A = R x_B + t, [12] R row-major | t); the state is M = T^-1, which moves A's samples into
B's frame."""
from __future__ import annotations

import math

import numpy as np

import distance_ref as dr
import grid_from_mesh_ref as gr
import track_ref as tr

f32, f64 = np.float32, np.float64
VALS = tr.VALS            # kTrackVals
AUX = 2                   # per system also sum w of the rows and a 0 (the device reports sum w for its first and last system only)
THREADS = 256             # kThreads: samples per block
DEFAULTS = dict(max_distance=(0.016, 0.008, 0.004), iterations=(10, 10, 10), samples_per_edge=1, min_normal_cos=0.5,
                min_correspondences=100)
IDENTITY = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]


def params(**over):
    p = dict(DEFAULTS)
    p.update(over)
    assert len(p["max_distance"]) == len(p["iterations"])
    p["max_distance"] = tuple(f32(d) for d in p["max_distance"])
    p["iterations"] = tuple(int(i) for i in p["iterations"])
    p["min_normal_cos"] = f32(p["min_normal_cos"])
    return p


def face_normals(mesh):
    """float32 unit face normal [F, 3]: n = (v1 - v0) x (v2 - v0) in dist_sample's operations, divided by __fsqrt_rn(dot(n, n)); 0 where
    that length is 0"""
    v = np.asarray(mesh["vertices"], f32)
    f = np.asarray(mesh["faces"], np.int64)
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], -1)
    ln = np.sqrt(dr._dot(n, n))
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(ln[:, None] > 0, n / np.where(ln > 0, ln, f32(1))[:, None], f32(0)).astype(f32)


def xform(Mf, v, translate=True):
    """tr_xform: R v (+ t) of the float pose Mf [12] on points v [N, 3], sums left to right"""
    out = tr.xform(Mf, Mf[9:] if translate else None, [v[:, 0], v[:, 1], v[:, 2]])
    return np.stack(out, -1).astype(f32)


def rows(A, B, M, L, max_distance, min_normal_cos, nA=None, nB=None):
    """The rows of every sample of A at the double pose M [12] (its float copy applied): dict with w [S] (0 for a row not kept), J [S, 6],
    r [S], kept [S], face [S] (the nearest face of B, -1 when unmatched or not queried) and the transformed samples p [S, 3]"""
    nA = face_normals(A) if nA is None else nA
    nB = face_normals(B) if nB is None else nB
    P, w = dr.samples(A, L)
    LL = L * L
    fa = np.repeat(np.arange(len(A["faces"])), LL)
    Mf = np.asarray(M, f64).astype(f32)
    p = xform(Mf, P)
    live = w > 0                                   # a zero-area face drops its samples
    face = np.full(len(P), -1, np.int32)
    if live.any():
        face[live] = dr.nearest(p[live], B, max_distance)[1]
    kept = face >= 0
    vb = np.asarray(B["vertices"], f32)
    fb = np.asarray(B["faces"], np.int64)
    k = np.flatnonzero(kept)
    c = np.zeros_like(p)
    if len(k):
        _, _, dv = gr.point_tri_feature(p[k], vb[fb[face[k], 0]], vb[fb[face[k], 1]], vb[fb[face[k], 2]])
        c[k] = p[k] - dv
    na = xform(Mf, nA[fa], translate=False)
    nb = np.where(kept[:, None], nB[np.maximum(face, 0)], f32(0))
    kept &= np.any(na != 0, axis=1) & np.any(nb != 0, axis=1)
    if min_normal_cos > f32(-1):
        kept &= dr._dot(na, nb) >= min_normal_cos
    pd, cd, nd = (np.where(kept[:, None], x, 0).astype(f64) for x in (p, c, nb))
    r = (nd[:, 0] * (pd[:, 0] - cd[:, 0]) + nd[:, 1] * (pd[:, 1] - cd[:, 1])) + nd[:, 2] * (pd[:, 2] - cd[:, 2])
    J = np.stack([pd[:, 1] * nd[:, 2] - pd[:, 2] * nd[:, 1], pd[:, 2] * nd[:, 0] - pd[:, 0] * nd[:, 2],
                  pd[:, 0] * nd[:, 1] - pd[:, 1] * nd[:, 0], nd[:, 0], nd[:, 1], nd[:, 2]], -1)
    return dict(w=np.where(kept, w, 0.0), J=J, r=r, kept=kept, face=face, p=p)


def values(R):
    """the VALS + AUX per-sample values: w J_a J_b (upper triangle, row by row), w J_a r, w r^2, 1 per row; then w, 0"""
    w, J, r, kept = R["w"], R["J"], R["r"], R["kept"]
    V = np.zeros((len(w), VALS + AUX), f64)
    wJ = w[:, None] * J
    for j, (a, b) in enumerate(tr.UPPER):
        V[:, j] = wJ[:, a] * J[:, b]
    for a in range(6):
        V[:, 21 + a] = wJ[:, a] * r
    V[:, 27] = (w * r) * r
    V[:, 28] = kept.astype(f64)
    V[:, VALS] = w
    return V


def block_sums(V):
    """the device's order: per block of 256 samples a shuffle-down tree over each warp and the 8 warps in order, then the blocks in order"""
    n, nv = V.shape
    nb = max(1, -(-n // THREADS))
    x = np.zeros((nb * THREADS, nv), f64)
    x[:n] = V
    x = x.reshape(nb, THREADS // 32, 32, nv)
    for o in (16, 8, 4, 2, 1):
        x[:, :, :o] = x[:, :, :o] + x[:, :, o:2 * o]
    w = x[:, :, 0]
    t = w[:, 0]
    for k in range(1, THREADS // 32):
        t = t + w[:, k]
    s = np.zeros(nv, f64)
    for b in range(nb):
        s = s + t[b]
    return s


def system(A, B, M, L, max_distance, min_normal_cos, nA=None, nB=None):
    """(the VALS + AUX sums, the rows) at pose M"""
    R = rows(A, B, M, L, max_distance, min_normal_cos, nA, nB)
    return block_sums(values(R)), R


def register(A, B, T_init=None, poses=None, **over):
    """i3d_register_reference_mesh restated.  Returns dict T (the final T [12]), status, iterations, update_norm, systems [E, VALS + AUX]
    (every system formed, the first at T_init, the last the solve-free one at the final pose), Ms [E, 12] (the pose M each was formed at).
    poses: [E, 12] M per system to use instead of the restatement's own (the device's, so that each system is checked on its own)."""
    p = params(**over)
    nA, nB = face_normals(A), face_normals(B)
    M = tr.inverse(IDENTITY if T_init is None else T_init)
    status, iterations, frozen, update_norm = 0, 0, False, 0.0
    systems, Ms = [], []
    sched = [(d, 1) for d, n in zip(p["max_distance"], p["iterations"]) for _ in range(n)] + [(p["max_distance"][-1], 0)]
    for e, (maxd, solve) in enumerate(sched):
        if poses is not None:
            M = [float(a) for a in poses[e]]
        S, _ = system(A, B, M, p["samples_per_edge"], maxd, p["min_normal_cos"], nA, nB)
        systems.append(S)
        Ms.append(list(M))
        if not solve or frozen:
            continue
        if int(S[28]) < p["min_correspondences"]:
            status, frozen = 1, True
            continue
        st, x = tr.solve(S[:VALS])
        if st:
            status, frozen = st, True
            continue
        Mn = tr.update(M, x)
        if not all(math.isfinite(a) for a in list(x) + Mn):
            status, frozen = 3, True
            continue
        M = Mn
        update_norm = math.sqrt(tr.sum_sq(x))
        iterations += 1
    return dict(T=np.array(tr.inverse(M)), M=np.array(M), status=status, iterations=iterations, update_norm=update_norm,
                systems=np.array(systems), Ms=np.array(Ms))


def summary(S):
    """(rows, sum w, sum w r^2, rms) of one system"""
    sw, sq = float(S[VALS]), float(S[27])
    return int(S[28]), sw, sq, math.sqrt(sq / sw) if sw > 0 else 0.0


def transform(vertices, T):
    """i3d_transform_reference_mesh: x <- float(((R0 x0 + R1 x1) + R2 x2) + t) per row, in double from the float x"""
    x = np.asarray(vertices, f32).astype(f64)
    T = np.asarray(T, f64)
    out = np.stack([((T[3 * i] * x[:, 0] + T[3 * i + 1] * x[:, 1]) + T[3 * i + 2] * x[:, 2]) + T[9 + i] for i in range(3)], -1)
    return out.astype(f32)


# ---- rigid motions for the tests and the benchmark ---------------------------------------------------------------------------------
def motion(rot_deg, trans, seed, centre=(0.0, 0.0, 0.0)):
    """[12] R | t in double: a rotation by rot_deg about a seeded axis through centre, then a translation of length trans in a seeded
    direction"""
    rng = np.random.default_rng(seed)
    a = rng.normal(size=3); a /= np.linalg.norm(a)
    d = rng.normal(size=3); d /= np.linalg.norm(d)
    th = math.radians(rot_deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K
    c = np.asarray(centre, f64)
    t = c - R @ c + trans * d
    return np.concatenate([R.reshape(-1), t])


def compose(A, B):
    """A . B of two [12] rigid motions"""
    Ra, Rb = np.asarray(A[:9]).reshape(3, 3), np.asarray(B[:9]).reshape(3, 3)
    return np.concatenate([(Ra @ Rb).reshape(-1), Ra @ np.asarray(B[9:]) + np.asarray(A[9:])])


def moved(mesh, G):
    """a copy of mesh with every vertex x -> G x in double, then rounded to float"""
    v = np.asarray(mesh["vertices"], f64)
    G = np.asarray(G, f64)
    return dict(vertices=(v @ G[:9].reshape(3, 3).T + G[9:]).astype(f32), faces=np.asarray(mesh["faces"], np.int32))


def errors(T, T_true, points):
    """(rotation error in degrees, largest displacement over points [N, 3] in metres) of T against T_true"""
    Ra, Rb = np.asarray(T[:9]).reshape(3, 3), np.asarray(T_true[:9]).reshape(3, 3)
    c = (np.trace(Ra @ Rb.T) - 1.0) * 0.5
    x = np.asarray(points, f64)
    d = x @ (Ra - Rb).T + (np.asarray(T[9:]) - np.asarray(T_true[9:]))
    return math.degrees(math.acos(min(1.0, max(-1.0, c)))), float(np.sqrt((d * d).sum(1)).max())
