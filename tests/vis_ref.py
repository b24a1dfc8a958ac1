"""Numpy float32 / float64 restatement of the mesh colour modes (DESIGN.md §6k), the checker of i3d_vis.cuh.

Written from the reference's SDFVisualization::applyColor* (libintrinsic3d/src/sdf/visualization.cpp:228-371), SDFOperators
(src/sdf/operators.cpp:58-139), Shading::computeShading (src/shading.cpp:61-73), Subvolumes::interpolate + math::average
(src/lighting/subvolumes.cpp:165-205, src/math.cpp:74-128) and color_util (src/color_util.cpp:41-78).  It shares no code with the kernels:
neighbours come from a sorted key table of the coordinates, not from the engine's neighbour table.  Every float32 operation is a numpy
float32 operation (rounded once, no fused multiply-add); every uchar cast truncates.
"""
import numpy as np

F32 = np.float32
MODES = ("", "normals", "lap", "lum", "lum_grad", "albedo", "shading_sv", "shading_sv_const", "chroma")
# +x, -x, +y, -y, +z, -z (SDFAlgorithms::collectRingNeighborhood)
RING = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.int64)
# math::interpolationWeights corner order
CORNERS = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0, 1, 1], [1, 0, 1], [1, 1, 1]], np.int64)


def _keys(c):
    c = np.asarray(c, np.int64) + (1 << 21)
    return (c[:, 0] << 44) | (c[:, 1] << 22) | c[:, 2]


class _Lookup:
    """coordinates -> row index, -1 where absent"""

    def __init__(self, coords):
        k = _keys(coords)
        self.order = np.argsort(k, kind="stable")
        self.sk = k[self.order]

    def __call__(self, q):
        k = _keys(q)
        if len(self.sk) == 0:
            return np.full(len(k), -1, np.int64)
        pos = np.clip(np.searchsorted(self.sk, k), 0, len(self.sk) - 1)
        return np.where(self.sk[pos] == k, self.order[pos], -1)


def scalar_to_color(v, scale=None):
    """scalarToColor(v, scale): min(max(v * scale, 0), 255), truncated (the multiply is left out for scale 1)."""
    if scale is not None:
        v = v * scale
    v = np.where(v < 0, v.dtype.type(0), v)
    v = np.where(v.dtype.type(255) < v, v.dtype.type(255), v)
    return np.trunc(v).astype(np.uint8)


def intensity(rgb):
    c = np.asarray(rgb, np.uint8).astype(F32)
    return (F32(0.299) * c[:, 0] + F32(0.587) * c[:, 1]) + F32(0.114) * c[:, 2]


def _grey(c):
    return np.repeat(np.asarray(c, np.uint8)[:, None], 3, axis=1)


def _ring(g):
    xyz = np.asarray(g["xyz"], np.int64)
    look = _Lookup(xyz)
    idx = np.stack([look(xyz + o) for o in RING], 1)
    w = np.asarray(g["weight"], np.float32)
    ok = np.where(idx >= 0, w[np.maximum(idx, 0)] > 0, False)
    return idx, ok


def surface_normals(sdf, weight, idx, ok):
    """computeSurfaceNormal in float32: (normal [n, 3], usable) where usable = the voxel and its +x/+y/+z neighbours are valid and the
    normal is neither zero nor NaN."""
    s = np.asarray(sdf, np.float64).astype(F32)
    usable = (np.asarray(weight, np.float32) > 0) & ok[:, 0] & ok[:, 2] & ok[:, 4]
    g = np.stack([s[np.maximum(idx[:, k], 0)] - s for k in (0, 2, 4)], 1)
    g = np.where(usable[:, None], g, F32(0))
    ln = np.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        n = np.where((ln != 0)[:, None], g / ln[:, None], g)
    usable &= ~((n == 0).all(1)) & ~np.isnan(n).any(1)
    return np.where(usable[:, None], n, F32(0)).astype(F32), usable


def blend_sh(xyz, voxel_size, sub_index, sub_sh, subvolume_size):
    """Subvolumes::interpolate(linear=true) of the subvolume SH at voxelToWorld of every voxel, in float64 (product and sum rounded
    separately), as float64 [n, 9]; zero where no surrounding subvolume exists."""
    xyz = np.asarray(xyz, np.int64)
    n = len(xyz)
    inv = F32(1) / F32(subvolume_size)
    pos = (xyz.astype(F32) * F32(voxel_size)) * inv - F32(0.5)
    fl = np.floor(pos)
    v0 = fl.astype(np.int64)
    wg = (pos - fl).astype(F32)
    look = _Lookup(np.asarray(sub_index, np.int64))
    sub_sh = np.asarray(sub_sh, np.float64)
    avg = np.zeros((n, 9), np.float64)
    sum_w = np.zeros(n, F32)
    for c in CORNERS:
        wx = np.where(c[0] == 1, wg[:, 0], F32(1) - wg[:, 0])
        wy = np.where(c[1] == 1, wg[:, 1], F32(1) - wg[:, 1])
        wz = np.where(c[2] == 1, wg[:, 2], F32(1) - wg[:, 2])
        w = ((wx * wy) * wz).astype(F32)
        sid = look(v0 + c)
        use = (sid >= 0) & (w != 0)
        prod = w.astype(np.float64)[:, None] * sub_sh[np.maximum(sid, 0)]
        first = (sum_w == 0)[:, None]
        avg = np.where(use[:, None], np.where(first, prod, avg + prod), avg)
        sum_w = np.where(use, sum_w + w, sum_w).astype(F32)
    nz = sum_w != 0
    with np.errstate(divide="ignore"):
        scale = (F32(1) / np.where(nz, sum_w, F32(1))).astype(np.float64)
    return np.where(nz[:, None], avg * scale[:, None], avg)


def shading(n, sh, albedo):
    """Shading::computeShading on unit normals: albedo * (sh . basis(n)) in float32, basis in Q9 order, the dot product summed
    k = 0..8 left to right; 0 where the albedo is 0 or NaN."""
    x, y, z = n[:, 0], n[:, 1], n[:, 2]
    b = [np.ones_like(x), y, z, x, x * y, y * z, ((-(x * x)) - (y * y)) + F32(2) * (z * z), x * z, (x * x) - (y * y)]
    d = sh[:, 0] * b[0]
    for k in range(1, 9):
        d = d + sh[:, k] * b[k]
    out = albedo * d
    return np.where((albedo == 0) | np.isnan(albedo), F32(0), out).astype(F32)


def colors(g, mode, source="refined", sub_index=None, sub_sh=None, subvolume_size=None):
    """Every voxel's colour in `mode` (a mode string of MODES), uint8 [n, 3].  g: the dict Engine.download_grid returns.  The shading
    modes take the subvolume indices [S, 3] and SH [S, 9] of a lighting estimate (Engine.download_lighting) and its subvolume size."""
    if mode not in MODES:
        raise ValueError(mode)
    rgb = np.asarray(g["rgb"], np.uint8)
    n = len(rgb)
    if mode == "":
        return rgb.copy()
    sdf = np.asarray(g["sdf_refined"] if source == "refined" else g["sdf0"], np.float64)
    idx, ok = _ring(g)
    ring_ok = ok.all(1)
    if mode == "normals":
        nrm, usable = surface_normals(sdf, g["weight"], idx, ok)
        c = scalar_to_color((F32(0.5) * nrm + F32(0.5)) * F32(255))
        return np.where(usable[:, None], c, np.uint8(0))
    if mode == "lap":
        s = sdf.astype(F32)
        d = [(s[np.maximum(idx[:, 2 * a], 0)] + s[np.maximum(idx[:, 2 * a + 1], 0)]) - F32(2) * s for a in range(3)]
        truncation = F32(g["voxel_size"]) * F32(5)
        lap = ((d[0] + d[1]) + d[2]) / truncation
        c = scalar_to_color(F32(0.5) * lap + F32(0.5), F32(255))
        return _grey(np.where(ring_ok, c, np.uint8(0)))
    if mode == "lum":
        return _grey(scalar_to_color(intensity(rgb)))
    if mode == "lum_grad":
        lum = intensity(rgb)
        dx = lum[np.maximum(idx[:, 0], 0)] - lum
        c = scalar_to_color(dx * F32(0.5) + F32(127))
        return _grey(np.where(ring_ok, c, np.uint8(127)))
    if mode == "albedo":
        return _grey(scalar_to_color(np.asarray(g["albedo"], np.float64), 255.0))
    if mode in ("shading_sv", "shading_sv_const"):
        nrm, usable = surface_normals(sdf, g["weight"], idx, ok)
        sub_sh = np.asarray(sub_sh, np.float64)
        if len(sub_sh) == 1:
            sh = np.repeat(sub_sh[:1].astype(F32), n, axis=0)
        else:
            sh = blend_sh(g["xyz"], g["voxel_size"], sub_index, sub_sh, subvolume_size).astype(F32)
        a = np.full(n, F32(0.7)) if mode == "shading_sv_const" else np.asarray(g["albedo"], np.float64).astype(F32)
        shad = (shading(nrm, sh, a).astype(np.float64) * 255.0).astype(F32)
        c = scalar_to_color(shad)
        return _grey(np.where(usable, c, np.uint8(0)))
    # chroma
    lum = intensity(rgb)
    inv = F32(1) / np.where(lum < F32(0.001), F32(0.001), lum)
    chrom = ((rgb.astype(F32) * inv[:, None]) * F32(255)) * F32(0.5)
    return scalar_to_color(chrom)
