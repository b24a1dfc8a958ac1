"""Float64 reference of the Gauss-Newton normal-equation kernels (k_eg_accum + k_acc_to_float + k_finish_problem, and the
CGNR operator k_eg_apply + k_op_partial), assembled as a scipy.sparse matrix from the rows the kernels themselves consumed.

Because the reference takes the kernels' own float inputs (float32 E_g Jacobian rows, the engine's row weights and Jacobi scale),
the only difference left between the two is the kernels' float arithmetic.  That is bounded componentwise, entry by entry:

    |x_gpu - x_ref|_j  <=  c * 2^-24 * M_j

where M_j is the same sum taken over absolute values (|J|, |r|, |v|) and c counts the float roundings on the longest chain of
the kernel that produces x (derivations at the constants below; first order: the neglected terms are O((c 2^-24)^2) relative).
Where the reference is structurally zero (fixed columns, frames no row sees) M_j = 0 and the kernel must give an exact zero.
"""
import numpy as np
import scipy.sparse as sp

U24 = 2.0 ** -24
# 10-voxel SDF stencil and 4 albedo neighbours of an E_g row, (x, y, z) offsets in the reference's parameter order
EG_SDF_OFFSETS = ((0, 0, 0), (0, 1, 0), (0, 2, 0), (0, 1, 1), (0, 0, 1), (0, 0, 2), (1, 0, 0), (1, 1, 0), (1, 0, 1), (2, 0, 0))
EG_ALB_OFFSETS = ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1))
FACE_OFFSETS = ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1))


def rounding_counts(K):
    """Float roundings on the longest chain of each quantity, K = observations per voxel.
    colnorm  c_j: voxel column: wf = float(w_raw), J*J, *wf (3) + K-1 adds of the per-thread sum + 1 for the double atomics
             + float(total) = K + 4.  Camera column: 3 products + 5 levels of the 32-lane reduce-scatter + block partial rounded
             to float + double atomics + float(total) = 11; intrinsics/distortion: 3 + K-1 adds + 5 + 3 = K + 10.  Max: K + 11.
    s  = float(1/(1+sqrt(c))): ds/s <= (dc/c)/2, + 1 for the rounding            -> c_nrm/2 + 1
    jtj = float(s^2 c) with the unrounded s: 2 (ds/s) + dc/c + 1                  -> 2 c_nrm + 1
    b  = float(s * w_g * grad): the gradient chain is the colnorm chain with wr = float(w_raw r) for wf, so <= c_nrm; + s + 1
    cam_acc (raw camera sums): the colnorm chain                                    -> c_nrm
    q  = s * float(float(qgd) + regulariser): u = J.ps with ps = float(s v) (1) over four FMA chains of <= 8 and 2 combining adds
         (11), wu = w u (1); voxel columns + K FMAs over the rows, double atomics (1), float(qgd), + regulariser, s * qg (3):
         K + 16; pose columns wu*J (1) + 5 shuffle levels + block partial + atomics + float(qgd) + s*qg = 22; intrinsics /
         distortion K FMAs + 5 levels + 4 = K + 21; E_r rows: ps, 7 + 7 adds of the two Laplacian gathers, float(w_r), w_r * t,
         2 adds into qg, s * qg = 20; E_a / E_s rows fewer.                          -> K + 21
    """
    c_nrm = K + 11
    return dict(colnorm=c_nrm, s=c_nrm / 2 + 1, jtj=2 * c_nrm + 1, b=c_nrm + c_nrm / 2 + 1, cam_acc=c_nrm, q=K + 21)


class VoxelIndex:
    """coordinates -> voxel index (the engine's neighbour table, restated on the host from xyz)"""

    def __init__(self, xyz):
        xyz = np.asarray(xyz, np.int64)
        self.lo = xyz.min(0) - 3
        self.ext = xyz.max(0) - self.lo + 4
        keys = self._key(xyz)
        self.order = np.argsort(keys)
        self.sorted = keys[self.order]
        self.xyz = xyz

    def _key(self, c):
        c = c - self.lo
        return (c[..., 2] * self.ext[1] + c[..., 1]) * self.ext[0] + c[..., 0]

    def lookup(self, vox, offset):
        """index of voxel vox + offset, -1 where it does not exist"""
        c = self.xyz[vox] + np.asarray(offset, np.int64)
        k = self._key(c)
        pos = np.clip(np.searchsorted(self.sorted, k), 0, len(self.sorted) - 1)
        found = self.sorted[pos] == k
        return np.where(found, self.order[pos], -1)


class Rows:
    """All rows of one iteration in unknown space [sdf n | albedo n | poses 6F | intr 4 | dist 5].
    Per row: up to 29 (column, raw Jacobian) entries, residual r, weight for the norms / gradient (w_raw * type weight, double)
    and weight of the operator (the float the kernels multiply with).  E_g rows also keep frame, raw weight and active slot."""

    def __init__(self, n, F):
        self.n, self.F = n, F
        self.U = 2 * n + 6 * F + 9
        self.cols, self.vals, self.res, self.w, self.w_op = [], [], [], [], []
        self.eg = None

    def add(self, cols, vals, res, w, w_op):
        self.cols.append(np.asarray(cols, np.int64))
        self.vals.append(np.asarray(vals, np.float64))
        self.res.append(np.asarray(res, np.float64))
        self.w.append(np.asarray(w, np.float64))
        self.w_op.append(np.asarray(w_op, np.float64))

    def matrix(self):
        """(J, r, w, w_op): J as CSR [rows x U]; entries on missing columns (-1) are dropped"""
        rows = [np.repeat(np.arange(c.shape[0]), c.shape[1]) for c in self.cols]
        off = np.cumsum([0] + [c.shape[0] for c in self.cols])
        ri = np.concatenate([r + o for r, o in zip(rows, off[:-1])])
        ci = np.concatenate([c.ravel() for c in self.cols])
        vi = np.concatenate([v.ravel() for v in self.vals])
        keep = (ci >= 0) & (vi != 0.0)
        J = sp.csr_matrix((vi[keep], (ri[keep], ci[keep])), shape=(int(off[-1]), self.U))
        return J, np.concatenate(self.res), np.concatenate(self.w), np.concatenate(self.w_op)


def eg_columns(idx, vox, frame, n, F):
    """[m, 29] unknown indices of E_g rows (voxel, frame), looked up from the coordinates"""
    m = len(vox)
    cols = np.empty((m, 29), np.int64)
    for c, off in enumerate(EG_SDF_OFFSETS):
        cols[:, c] = idx.lookup(vox, off)
    for c, off in enumerate(EG_ALB_OFFSETS):
        nb = idx.lookup(vox, off)
        cols[:, 10 + c] = np.where(nb >= 0, n + nb, -1)
    cols[:, 14:20] = 2 * n + 6 * np.asarray(frame, np.int64)[:, None] + np.arange(6)
    cols[:, 20:29] = 2 * n + 6 * F + np.arange(9)
    return cols


def build_rows(scene, eg, reg, type_w):
    """eg: dict voxel, frame, residual, raw_weight, J [m, 29] (float64), w_op [m], slot [m] (active index of the voxel).
    reg: the oracle's rows(1), rows(2), rows(3) (E_r, E_s, E_a).  type_w: the iteration's four type weights (double)."""
    xyz = scene["xyz"]
    n, F = xyz.shape[0], scene["poses"].shape[0]
    idx = VoxelIndex(xyz)
    R = Rows(n, F)
    vox = np.asarray(eg["voxel"], np.int64)
    cols = eg_columns(idx, vox, eg["frame"], n, F)
    assert (cols[:, :14] >= 0).all(), "E_g row with an incomplete stencil"
    R.add(cols, eg["J"], eg["residual"], eg["raw_weight"] * type_w[0], eg["w_op"])
    R.eg = dict(frame=np.asarray(eg["frame"], np.int64), raw_weight=np.asarray(eg["raw_weight"], np.float64),
                residual=np.asarray(eg["residual"], np.float64), J=np.asarray(eg["J"], np.float64),
                slot=np.asarray(eg.get("slot", np.zeros(len(vox))), np.int64), m=len(vox))
    f32 = lambda x: np.float64(np.float32(x))
    r1, r2, r3 = reg
    if len(r1["voxel"]):
        v = np.asarray(r1["voxel"], np.int64)
        c = np.stack([v] + [idx.lookup(v, o) for o in FACE_OFFSETS], 1)
        assert (c >= 0).all()
        J = np.tile(np.array([-6.0, 1, 1, 1, 1, 1, 1]), (len(v), 1))
        R.add(c, J, r1["residual"], r1["raw_weight"] * type_w[1], f32(type_w[1]) * r1["raw_weight"])
    if len(r2["voxel"]):
        v = np.asarray(r2["voxel"], np.int64)
        jac = (scene["sdf_refined"][v] != scene["sdf0"][v]).astype(np.float64)      # a residual pinned to 1e-7 has no derivative
        R.add(v[:, None], jac[:, None], r2["residual"], r2["raw_weight"] * type_w[2], f32(type_w[2]) * r2["raw_weight"])
    if len(r3["voxel"]):
        v = np.asarray(r3["voxel"], np.int64)
        b = np.asarray(r3["aux"], np.int64)
        R.add(np.stack([n + v, n + b], 1), np.tile(np.array([1.0, -1.0]), (len(v), 1)), r3["residual"],
              r3["raw_weight"] * type_w[3], f32(type_w[3]) * f32(r3["raw_weight"]))
    return R


class Perturb:
    """Deliberate errors for the comparator's own test: rows removed, extra multiples of some E_g rows' pose contributions,
    one column scaled."""

    def __init__(self, drop_eg_row=None, pose_extra=None, col_scale=None):
        self.drop_eg_row, self.pose_extra, self.col_scale = drop_eg_row, pose_extra, col_scale


def evaluate(R, free, s_op, vs=(), perturb=None):
    """Reference values and magnitude sums.  free: bool [U]; s_op: the Jacobi scale the operator is applied with (the engine's);
    vs: input vectors of the operator.  Returns {name: (ref, magnitude)} for colnorm, s, jtj, b, cam_acc and q0, q1, ..."""
    J, r, w, w_op = R.matrix()
    m_eg = R.eg["m"]
    if perturb is not None and perturb.col_scale is not None:
        j, f = perturb.col_scale
        d = np.ones(R.U)
        d[j] = f
        J = (J @ sp.diags(d)).tocsr()
    keep = np.ones(J.shape[0], bool)
    if perturb is not None and perturb.drop_eg_row is not None:
        keep[perturb.drop_eg_row] = False
    J, r, w, w_op = J[keep], r[keep], w[keep], w_op[keep]
    eg_keep = keep[:m_eg]
    # output-side copy of J: the rows' contributions as the kernels would ADD them (a double-added partial = extra multiple)
    Jout = J
    if perturb is not None and perturb.pose_extra is not None:
        rows, mult = perturb.pose_extra
        lo, hi = 2 * R.n, 2 * R.n + 6 * R.F
        D = J[rows].tocoo()
        sel = (D.col >= lo) & (D.col < hi)
        extra = sp.csr_matrix((D.data[sel] * mult, (np.asarray(rows)[D.row[sel]], D.col[sel])), shape=J.shape)
        Jout = (J + extra).tocsr()
    A = abs(J)
    Aout = abs(Jout)
    out = {}
    JJ = Jout.multiply(J).tocsr()
    c = JJ.T @ w
    cm = abs(JJ).T @ w
    s_ref = np.where(free, 1.0 / (1.0 + np.sqrt(c)), 0.0)
    out["colnorm"] = (c, cm)
    out["s"] = (s_ref, s_ref)
    out["jtj"] = (s_ref * s_ref * c, s_ref * s_ref * cm)
    out["b"] = (s_ref * (Jout.T @ (w * r)), s_ref * (Aout.T @ (w * np.abs(r))))
    m_kept = int(eg_keep.sum())          # the E_g rows come first
    out["cam_acc"] = cam_sums(R, Jout[:m_kept], J[:m_kept], R.eg["raw_weight"][eg_keep], R.eg["residual"][eg_keep], R.eg["frame"][eg_keep])
    s_op = np.asarray(s_op, np.float64)
    for i, v in enumerate(vs):
        v = np.asarray(v, np.float64)
        u = J @ (s_op * v)
        um = A @ (s_op * np.abs(v))
        out[f"q{i}"] = (s_op * (Jout.T @ (w_op * u)), s_op * (Aout.T @ (w_op * um)))
    return out


def cam_sums(R, Jout, J, w_raw, res, frame):
    """CamAccLayout of the raw E_g camera sums: per frame 6 gradient, 6 column norms, 21 upper 6x6; then 9 gradient, 9 column norms,
    10 + 15 upper triangles of intrinsics / distortion.  Returns (value, magnitude), each [33F + 43]."""
    n, F = R.n, R.F
    m = J.shape[0]
    P = _rows_cols(J, 2 * n + 6 * frame[:, None] + np.arange(6))
    Po = _rows_cols(Jout, 2 * n + 6 * frame[:, None] + np.arange(6))
    T = _rows_cols(J, np.broadcast_to(2 * n + 6 * F + np.arange(9), (m, 9)))
    To = _rows_cols(Jout, np.broadcast_to(2 * n + 6 * F + np.arange(9), (m, 9)))
    val = np.zeros(33 * F + 43)
    mag = np.zeros(33 * F + 43)
    wr = w_raw * res
    tri6 = [(a, b) for a in range(6) for b in range(a, 6)]

    def put(k, x, xm):
        val[k::33][:F] += np.bincount(frame, x, F)
        mag[k::33][:F] += np.bincount(frame, xm, F)

    for c in range(6):
        put(c, wr * Po[:, c], np.abs(wr * Po[:, c]))
        put(6 + c, w_raw * Po[:, c] * P[:, c], np.abs(w_raw * Po[:, c] * P[:, c]))
    for t, (a, b) in enumerate(tri6):
        put(12 + t, w_raw * Po[:, a] * P[:, b], np.abs(w_raw * Po[:, a] * P[:, b]))
    tail = 33 * F
    for c in range(9):
        val[tail + c] = np.sum(wr * To[:, c]); mag[tail + c] = np.sum(np.abs(wr * To[:, c]))
        val[tail + 9 + c] = np.sum(w_raw * To[:, c] * T[:, c]); mag[tail + 9 + c] = np.sum(np.abs(w_raw * To[:, c] * T[:, c]))
    t = tail + 18
    for lo, d in ((0, 4), (4, 5)):
        for a in range(d):
            for b in range(a, d):
                x = w_raw * To[:, lo + a] * T[:, lo + b]
                val[t] = x.sum(); mag[t] = np.abs(x).sum(); t += 1
    return val, mag


def _rows_cols(M, cols):
    """M[i, cols[i, k]] for every row i (dense [m, k]); M is CSR with at most 29 entries per row"""
    M = sp.csr_matrix(M)
    m = M.shape[0]
    out = np.zeros(cols.shape)
    rows = np.repeat(np.arange(m), np.diff(M.indptr))
    # position of each stored entry among the wanted columns of its row
    for k in range(cols.shape[1]):
        hit = M.indices == cols[rows, k]
        out[rows[hit], k] = M.data[hit]
    return out


def compare(gpu, ref, c):
    """(max over j of |gpu - ref| / (c 2^-24 M_j), every entry within its bound, number outside); M_j = 0 requires an exact zero"""
    val, mag = ref
    gpu = np.asarray(gpu, np.float64)
    err = np.abs(gpu - val)
    bound = c * U24 * mag
    ok = err <= bound
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(ratio.max()) if ratio.size else 0.0, bool(ok.all()), int((~ok).sum())
