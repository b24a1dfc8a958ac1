"""Numpy restatement of the mesh simplification by quadric-error vertex clustering (DESIGN.md §6s), the checker of the k_simp_* kernels.

Lindstrom 2000, "Out-of-core simplification of large polygonal models", over a mesh dict as Engine.extract_mesh returns it (vertices
float32 [V, 3], colors uint8 [V, 3], faces int32 [F, 3]).  Written from the contract, sharing no code with the kernels: clusters come
from np.unique, duplicates from np.unique over the rotation keys, and every per-cluster sum runs over clusters at once, one member
rank at a time, so each cluster's sum is sequential in member order exactly as one device thread sums it.  Every float64 operation
below is one IEEE operation in the order written; numpy contracts nothing into an FMA.

Order of the arithmetic (double unless said otherwise):
  cell        floor(float32(x) / float32(cell)) in float32, per axis; refused unless finite and in [-2^31, 2^31)
  face        v0, v1, v2 widened from float32; e1 = v1 - v0, e2 = v2 - v0;
              n = (e1y*e2z - e1z*e2y, e1z*e2x - e1x*e2z, e1x*e2y - e1y*e2x); a = sqrt((nx*nx + ny*ny) + nz*nz);
              a == 0 or not finite: the face adds zeros.  u = n / a (each component); d = -((ux*v0x + uy*v0y) + uz*v0z);
              A_ij = (a*u_i)*u_j for (xx, xy, xz, yy, yz, zz); b_i = (a*d)*u_i.  (c = (a*d)*d does not move the minimiser: not summed.)
  cluster     A, b: 0 + q(first corner) + q(next corner) ... over the cluster's corners 3f + k in increasing order;
              position sum: 0 + x(first member) + ... over the members in vertex-id order; mean = sum / n
  solve       r_i = -b_i - ((A_i0*m0 + A_i1*m1) + A_i2*m2) with the summed A; cyclic Jacobi on A (jacobi3); y_j = ((V0j*r0 + V1j*r1) + V2j*r2),
              then y_j / l_j if l_j > 0 and l_j >= 1e-3 * max(l) else 0; x_i = float32(m_i + ((Vi0*y0 + Vi1*y1) + Vi2*y2)); the float32 mean
              when any x_i is not finite; a single-member cluster keeps its vertex
  colour      (sum + n // 2) // n per channel, in integers
"""
import numpy as np

import mesh_ref

F32, F64 = np.float32, np.float64
JACOBI_SWEEPS = 8
EIGEN_CUT = 1e-3
PAIRS = ((0, 1), (0, 2), (1, 2))
# the counts of I3DSimplifyInfo, in its order
INFO_COUNTS = ("num_clusters", "num_faces_collapsed", "num_faces_duplicate", "num_faces_degenerate", "num_faces", "num_vertices")


def jacobi3(a):
    """Cyclic Jacobi of symmetric 3x3 matrices a [..., 3, 3] (float64): (eigenvalues [..., 3], eigenvectors [..., 3, 3] as columns).
    Pairs (0,1), (0,2), (1,2) per sweep, JACOBI_SWEEPS sweeps; a pair whose off-diagonal entry is exactly 0 is left alone.
    tau = (a_qq - a_pp) / (2 a_pq), t = sgn(tau) / (|tau| + sqrt(1 + tau^2)) (sgn(0) = 1), c = 1 / sqrt(1 + t^2), s = t c;
    a_pp -= t a_pq, a_qq += t a_pq, a_pq = 0, a_rp = c a_rp - s a_rq, a_rq = s a_rp + c a_rq, and the same on the columns of V."""
    m = np.array(a, F64, copy=True)
    v = np.broadcast_to(np.eye(3), m.shape).copy()
    with np.errstate(all="ignore"):
        for _ in range(JACOBI_SWEEPS):
            for p, q in PAIRS:
                r = 3 - p - q
                apq = m[..., p, q].copy()
                go = apq != 0.0
                tau = (m[..., q, q] - m[..., p, p]) / (2.0 * apq)
                t = np.where(tau < 0.0, -1.0, 1.0) / (np.abs(tau) + np.sqrt(1.0 + tau * tau))
                c = 1.0 / np.sqrt(1.0 + t * t)
                s = t * c
                app = m[..., p, p] - t * apq
                aqq = m[..., q, q] + t * apq
                arp, arq = m[..., r, p].copy(), m[..., r, q].copy()
                nrp = c * arp - s * arq
                nrq = s * arp + c * arq
                m[..., p, p] = np.where(go, app, m[..., p, p])
                m[..., q, q] = np.where(go, aqq, m[..., q, q])
                m[..., p, q] = m[..., q, p] = np.where(go, 0.0, apq)
                m[..., r, p] = m[..., p, r] = np.where(go, nrp, arp)
                m[..., r, q] = m[..., q, r] = np.where(go, nrq, arq)
                for k in range(3):
                    vp, vq = v[..., k, p].copy(), v[..., k, q].copy()
                    v[..., k, p] = np.where(go, c * vp - s * vq, vp)
                    v[..., k, q] = np.where(go, s * vp + c * vq, vq)
    return np.stack([m[..., 0, 0], m[..., 1, 1], m[..., 2, 2]], -1), v


def cells(vertices, cell_size):
    """Integer cell of every vertex, int64 [V, 3]; raises ValueError when a quotient is not finite or outside int32."""
    with np.errstate(all="ignore"):
        q = np.floor(np.asarray(vertices, F32) / F32(cell_size))
    if not (np.isfinite(q).all() and (q >= F32(-2.0 ** 31)).all() and (q < F32(2.0 ** 31)).all()):
        raise ValueError("a cell coordinate is not finite or outside int32")
    return q.astype(np.int64)


def face_quadrics(vertices, faces):
    """Per face A (xx, xy, xz, yy, yz, zz) and b (x, y, z), float64 [F, 9], in the order of the module docstring."""
    P = np.asarray(vertices, F32).astype(F64)
    v0, v1, v2 = P[faces[:, 0]], P[faces[:, 1]], P[faces[:, 2]]
    e1, e2 = v1 - v0, v2 - v0
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    with np.errstate(all="ignore"):
        a = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
        ok = (a != 0.0) & np.isfinite(a)
        u = n / a[:, None]
        d = -((u[:, 0] * v0[:, 0] + u[:, 1] * v0[:, 1]) + u[:, 2] * v0[:, 2])
        wu = a[:, None] * u
        wd = a * d
        q = np.stack([wu[:, 0] * u[:, 0], wu[:, 0] * u[:, 1], wu[:, 0] * u[:, 2], wu[:, 1] * u[:, 1], wu[:, 1] * u[:, 2], wu[:, 2] * u[:, 2],
                      wd * u[:, 0], wd * u[:, 1], wd * u[:, 2]], 1)
    return np.where(ok[:, None], q, 0.0)


def _ranked_sum(values, group, n_groups):
    """Per group, 0 + values of its first item + values of its next item ..., items in their given order: float64 [n_groups, ...].
    Vectorised over the groups, one rank at a time."""
    order = np.argsort(group, kind="stable")
    cnt = np.bincount(group, minlength=n_groups)
    start = np.cumsum(cnt) - cnt
    by_cnt = np.argsort(-cnt, kind="stable")
    neg_sorted = -cnt[by_cnt]
    acc = np.zeros((n_groups,) + values.shape[1:], F64)
    for r in range(int(cnt.max()) if n_groups else 0):
        g = by_cnt[:np.searchsorted(neg_sorted, -r, side="left")]       # the groups with more than r items
        acc[g] = acc[g] + values[order[start[g] + r]]
    return acc


def _rotation_keys(f):
    """The rotation of each face that puts the smallest id first (for faces with three distinct ids)."""
    r1, r2 = np.roll(f, -1, 1), np.roll(f, -2, 1)
    a, b, c = f[:, 0], f[:, 1], f[:, 2]
    use1 = (b < a) & (b <= c)
    use2 = ~use1 & (c < a) & (c < b)
    return np.where(use1[:, None], r1, np.where(use2[:, None], r2, f))


def simplify(mesh, cell_size):
    """The simplified mesh dict (vertices, colors, faces, info: the counts of I3DSimplifyInfo)."""
    V = np.asarray(mesh["vertices"], F32).reshape(-1, 3)
    C = np.asarray(mesh["colors"], np.uint8).reshape(-1, 3)
    Fc = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    nv, nf = len(V), len(Fc)
    # 1. clusters by first appearance over the vertex ids
    if nv:
        cl = cells(V, cell_size)
        _, first, inv = np.unique(cl, axis=0, return_index=True, return_inverse=True)
        inv = inv.reshape(-1)
        by_first = np.argsort(first, kind="stable")
        rank = np.empty(len(first), np.int64)
        rank[by_first] = np.arange(len(first))
        cid = rank[inv]
        first_vertex = first[by_first]                       # per cluster, its lowest vertex id
    else:
        cid = first_vertex = np.zeros(0, np.int64)
    K = int(cid.max()) + 1 if nv else 0
    info = dict(num_clusters=K, num_faces_collapsed=0, num_faces_duplicate=0, num_faces_degenerate=0)
    empty = dict(vertices=np.zeros((0, 3), F32), colors=np.zeros((0, 3), np.uint8), faces=np.zeros((0, 3), np.int32))
    if nf == 0:
        info.update(num_faces=0, num_vertices=0)
        return dict(**empty, info=info)
    # 2., 3. quadrics and member sums, per cluster in order
    Q = _ranked_sum(face_quadrics(V, Fc)[np.arange(3 * nf) // 3], cid[Fc.reshape(-1)], K)
    S = _ranked_sum(V.astype(F64), cid, K)
    n = np.bincount(cid, minlength=K)
    csum = np.zeros((K, 3), np.int64)
    np.add.at(csum, cid, C.astype(np.int64))
    # 4. representatives
    with np.errstate(all="ignore"):
        mean = S / n[:, None].astype(F64)
        A = np.stack([np.stack([Q[:, 0], Q[:, 1], Q[:, 2]], -1), np.stack([Q[:, 1], Q[:, 3], Q[:, 4]], -1),
                      np.stack([Q[:, 2], Q[:, 4], Q[:, 5]], -1)], 1)
        r = -Q[:, 6:9] - ((A[:, :, 0] * mean[:, 0:1] + A[:, :, 1] * mean[:, 1:2]) + A[:, :, 2] * mean[:, 2:3])
        lam, vec = jacobi3(A)
        lmax = np.fmax(np.fmax(lam[:, 0], lam[:, 1]), lam[:, 2])
        cut = EIGEN_CUT * lmax
        y = (vec[:, 0, :] * r[:, 0:1] + vec[:, 1, :] * r[:, 1:2]) + vec[:, 2, :] * r[:, 2:3]
        y = np.where((lam > 0.0) & (lam >= cut[:, None]), y / lam, 0.0)
        dx = (vec[:, :, 0] * y[:, 0:1] + vec[:, :, 1] * y[:, 1:2]) + vec[:, :, 2] * y[:, 2:3]
        x = (mean + dx).astype(F32)
    ok = np.isfinite(x).all(1)
    rep = np.where(ok[:, None], x, mean.astype(F32))
    single = n == 1
    rep[single] = V[first_vertex[single]]
    rcol = ((csum + (n // 2)[:, None]) // n[:, None]).astype(np.uint8)
    # 5. faces: collapsed, duplicate (first occurrence kept), then the degenerate-face predicate at the representatives
    cf = cid[Fc]
    collapsed = (cf[:, 0] == cf[:, 1]) | (cf[:, 0] == cf[:, 2]) | (cf[:, 1] == cf[:, 2])
    live = np.nonzero(~collapsed)[0]
    dup = np.zeros(nf, bool)
    if len(live):
        _, firstk = np.unique(_rotation_keys(cf[live]), axis=0, return_index=True)
        keep_first = np.zeros(len(live), bool)
        keep_first[firstk] = True
        dup[live[~keep_first]] = True
    out = mesh_ref.clean(rep, cf[~dup])                      # drops the collapsed faces too (repeated indices); keeps the order
    info.update(num_faces_collapsed=int(collapsed.sum()), num_faces_duplicate=int(dup.sum()),
                num_faces_degenerate=int(nf - len(out) - collapsed.sum() - dup.sum()))
    # 6. only the clusters the faces use, in order
    used = np.zeros(K, bool)
    used[out.ravel()] = True
    new_id = np.cumsum(used) - 1
    faces = new_id[out].astype(np.int32).reshape(-1, 3)
    info.update(num_faces=len(faces), num_vertices=int(used.sum()))
    return dict(vertices=rep[used], colors=rcol[used], faces=faces, info=info)
