"""CPU checks of the RGB-D fusion oracle (tests/native/fusion_oracle.cpp), the checker of the device fusion kernels:
KF1 an independent numpy-float32 restatement reproduces it exactly; KF2 synthetic truth; KF3 correctSDF properties; KF4 allocation
properties; and the golden fixture."""
import os

import numpy as np
import pytest

from fusion_ref import FusionOracle, bounds, depth_range, erode, normals, scene_inputs

f32 = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))


def _scene(frames=3):
    from intrinsic3d_b200.scene import make_scene
    return make_scene(radius_vox=10.0, frames=frames, width=96, height=72, voxel_size=0.004, seed=2)


def _okw(s, window=2, ws=10.0, clip=(0.0,) * 6):
    dmin, dmax = depth_range(s)
    return dict(voxel_size=float(s["voxel_size"]), depth_min=dmin, depth_max=dmax, weight_sample=ws, clip=clip, window=window, iterations=10)


# ---------------------------------------------------------------- numpy float32 restatement (KF1)
def np_erode(d, w):
    if w <= 0:
        return d.copy()
    H, W = d.shape
    out = d.copy()
    for y in range(H):
        for x in range(W):
            r = d[y, x]
            if r == 0:
                continue
            win = d[max(0, y - w):min(y + w, H - 1) + 1, max(0, x - w):min(x + w, W - 1) + 1]
            if (win == 0).any() or (np.abs(win - r) > f32(0.5)).any():
                out[y, x] = 0
    return out


def np_normals(cam, d):
    W, H, fx, fy, cx, cy = (f32(v) for v in cam)
    H, W = d.shape
    x0 = (np.arange(W, dtype=f32) - cx) * (f32(1) / fx)
    y0 = (np.arange(H, dtype=f32) - cy) * (f32(1) / fy)
    v = np.stack([x0[None, :] * d, y0[:, None] * d, d], -1)
    tx = v[1:-1, 2:] - v[1:-1, :-2]
    ty = v[2:, 1:-1] - v[:-2, 1:-1]
    nrm = lambda a: np.sqrt((a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1]) + a[..., 2] * a[..., 2])
    ok = (d[1:-1, 1:-1] != 0) & (d[1:-1, :-2] != 0) & (d[1:-1, 2:] != 0) & (d[:-2, 1:-1] != 0) & (d[2:, 1:-1] != 0)
    ok &= (nrm(tx) < f32(0.3)) & (nrm(ty) < f32(0.3))
    c = np.stack([ty[..., 1] * tx[..., 2] - ty[..., 2] * tx[..., 1], ty[..., 2] * tx[..., 0] - ty[..., 0] * tx[..., 2],
                  ty[..., 0] * tx[..., 1] - ty[..., 1] * tx[..., 0]], -1)
    sq = (c[..., 0] * c[..., 0] + c[..., 1] * c[..., 1]) + c[..., 2] * c[..., 2]
    with np.errstate(invalid="ignore", divide="ignore"):
        cn = np.where((sq > 0)[..., None], c / np.sqrt(sq)[..., None], c)
    out = np.zeros(d.shape + (3,), f32)
    out[1:-1, 1:-1] = np.where(ok[..., None], cn, f32(0))
    return out


def xf(R, t, p):
    """R [9], t [3] float32; p [..., 3] -> left-to-right sums."""
    return np.stack([((R[3 * k] * p[..., 0] + R[3 * k + 1] * p[..., 1]) + R[3 * k + 2] * p[..., 2]) + t[k] for k in range(3)], -1)


def w2v(p, inv):
    return (p * inv + f32(0.5)).astype(np.int32)


def np_bounds(cam, dmin, dmax, vs, rt):
    W, H, fx, fy, cx, cy = cam
    inv = f32(1) / f32(vs)
    pts = []
    for d in (dmin, dmax):
        for u, v in ((0, 0), (W - 1, 0), (W - 1, H - 1), (0, H - 1)):
            d = f32(d)
            pts.append([d * ((f32(u) - f32(cx)) / f32(fx)), d * ((f32(v) - f32(cy)) / f32(fy)), d] if d != 0 else [f32(0)] * 3)
    p = xf(rt[:9], rt[9:], np.array(pts, f32))
    lo, hi = w2v(np.floor(p), inv), w2v(np.ceil(p), inv)
    allv = np.concatenate([lo, hi])
    return np.array([allv[:, 0].min(), allv[:, 0].max(), allv[:, 1].min(), allv[:, 1].max(), allv[:, 2].min(), allv[:, 2].max()], np.int32)


def np_fuse(s, kw, frames):
    """Allocation + integration of `frames` frames; returns {packed coordinate: [sdf, weight, r, g, b]} as float32 arrays."""
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    vs = f32(kw["voxel_size"]); trunc = vs * f32(5); step = vs * f32(0.25); inv = f32(1) / vs
    clip = np.array(kw["clip"], f32); use_clip = float((clip * clip).sum()) > 0
    W, H, fx, fy, cx, cy = (f32(v) for v in dcam)
    W, H = int(W), int(H)
    coords = np.zeros((0, 3), np.int64); sdf = np.zeros(0, f32); wt = np.zeros(0, f32); col = np.zeros((0, 3), np.uint8)
    ws = f32(kw["weight_sample"])
    for f in range(frames):
        d = np_erode(depth[f], kw["window"])
        nm = np_normals(dcam, d)
        b = np_bounds(dcam, kw["depth_min"], kw["depth_max"], kw["voxel_size"], c2w[f])
        ys, xs = np.nonzero(d)
        dd = d[ys, xs]
        pc = np.stack([(xs.astype(f32) - cx) / fx, (ys.astype(f32) - cy) / fy, np.ones(len(xs), f32)], -1)
        last = np.zeros((len(xs), 3), np.int32)
        cent = []
        d_off = -trunc
        while d_off <= trunc:
            g = w2v(xf(c2w[f, :9], c2w[f, 9:], pc * (dd + d_off)[:, None]), inv)
            new = (g != last).any(1)
            last = np.where(new[:, None], g, last)
            ok = new & (g[:, 0] >= b[0]) & (g[:, 0] <= b[1]) & (g[:, 1] >= b[2]) & (g[:, 1] <= b[3]) & (g[:, 2] >= b[4]) & (g[:, 2] <= b[5])
            if use_clip:
                pw = g.astype(f32) * vs
                ok &= ~((pw[:, 0] < clip[0]) | (pw[:, 0] > clip[1]) | (pw[:, 1] < clip[2]) | (pw[:, 1] > clip[3]) | (pw[:, 2] < clip[4]) | (pw[:, 2] > clip[5]))
            cent.append(g[ok])
            d_off = f32(d_off + step)
        cent = np.unique(np.concatenate(cent), axis=0).astype(np.int64)
        off = np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3)
        blk = np.unique((cent[:, None, :] + off[None]).reshape(-1, 3), axis=0)
        known = {tuple(c) for c in coords.tolist()}
        add = np.array([c for c in blk.tolist() if tuple(c) not in known], np.int64).reshape(-1, 3)
        coords = np.concatenate([coords, add]); sdf = np.concatenate([sdf, np.zeros(len(add), f32)])
        wt = np.concatenate([wt, np.zeros(len(add), f32)]); col = np.concatenate([col, np.zeros((len(add), 3), np.uint8)])
        # integrate
        inb = (coords[:, 0] >= b[0]) & (coords[:, 0] <= b[1]) & (coords[:, 1] >= b[2]) & (coords[:, 1] <= b[3]) & (coords[:, 2] >= b[4]) & (coords[:, 2] <= b[5])
        p = xf(w2c[f, :9], w2c[f, 9:], coords.astype(f32) * vs)
        with np.errstate(all="ignore"):
            u = (((p[:, 0] * fx) / p[:, 2] + cx) + f32(0.5)); v = (((p[:, 1] * fy) / p[:, 2] + cy) + f32(0.5))
            u = np.where(np.isfinite(u), u, f32(-1e9)).clip(-1e9, 1e9).astype(np.int64); v = np.where(np.isfinite(v), v, f32(-1e9)).clip(-1e9, 1e9).astype(np.int64)
        ok = inb & (p[:, 2] >= 0) & (u >= 0) & (v >= 0) & (u < W) & (v < H)
        i = np.nonzero(ok)[0]
        dv = d[v[i], u[i]]
        i = i[dv > 0]; dv = d[v[i], u[i]]
        pp = p[i]
        sd = dv - pp[:, 2]
        keep = sd > -trunc
        i, dv, pp, sd = i[keep], dv[keep], pp[keep], sd[keep]
        ts = np.where(sd >= 0, np.minimum(trunc, sd), np.maximum(-trunc, sd))
        wu = np.ones(len(i), f32)
        if ws > 0:
            n = nm[v[i], u[i]]
            sq = (pp[:, 0] * pp[:, 0] + pp[:, 1] * pp[:, 1]) + pp[:, 2] * pp[:, 2]
            q = np.where((sq > 0)[:, None], pp / np.sqrt(sq)[:, None], pp)
            rk = lambda x: f32(1) / (((f32(1) + f32(2) * x) * (f32(1) + f32(2) * x)) * (f32(1) + f32(2) * x))
            wn = f32(1) - np.abs((q[:, 0] * n[:, 0] + q[:, 1] * n[:, 1]) + q[:, 2] * n[:, 2])
            wn = np.maximum(np.minimum(wn, f32(1)), f32(0))
            wn = np.maximum(ws * rk(wn), f32(1))
            wd = np.maximum(ws * rk((f32(2) * np.abs(ts)) / trunc), f32(1))
            dn = (dv - f32(kw["depth_min"])) / (f32(kw["depth_max"]) - f32(kw["depth_min"]))
            wz = np.maximum(ws * (f32(1) - dn), f32(1))
            wu = np.maximum(((wn + wd) + wz) / f32(3), f32(3))
        wo = wt[i]; wnw = wo + wu
        sdf[i] = (sdf[i] * wo + sd * wu) / wnw
        CW, CH, cfx, cfy, ccx, ccy = (f32(x) for x in ccam)
        cu = (((pp[:, 0] * cfx) / pp[:, 2] + ccx) + f32(0.5)).astype(np.int64); cv = (((pp[:, 1] * cfy) / pp[:, 2] + ccy) + f32(0.5)).astype(np.int64)
        inc = (cu >= 0) & (cv >= 0) & (cu < int(CW)) & (cv < int(CH))
        j = i[inc]
        cn = bgr[f][cv[inc], cu[inc]][:, ::-1].astype(f32)
        col[j] = ((col[j].astype(f32) * wo[inc][:, None] + cn * wu[inc][:, None]) / wnw[inc][:, None]).astype(np.int32).astype(np.uint8)
        wt[i] = wnw
    return coords, sdf, wt, col


def _canon(xyz):
    c = (xyz.astype(np.int64) + (1 << 20)).astype(np.uint64)
    s3, s7 = np.uint64(3), np.uint64(7)
    key = ((c[:, 2] >> s3) << np.uint64(46)) | ((c[:, 1] >> s3) << np.uint64(28)) | ((c[:, 0] >> s3) << np.uint64(10)) | ((c[:, 2] & s7) << np.uint64(6)) \
        | ((c[:, 1] & s7) << s3) | (c[:, 0] & s7)
    return np.argsort(key, kind="stable")


@pytest.mark.parametrize("window,ws", [(0, 0.0), (2, 0.0), (0, 10.0), (2, 10.0)])
def test_kf1_numpy_restatement_matches_oracle(window, ws):
    s = _scene(frames=3)
    kw = _okw(s, window=window, ws=ws)
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    # pieces: erosion, normals, bounds
    for f in range(2):
        e = erode(depth[f], window)
        assert np.array_equal(e, np_erode(depth[f], window))
        assert np.array_equal(normals(dcam, e).view(np.uint32), np_normals(dcam, e).view(np.uint32))
        assert np.array_equal(bounds(dcam, kw["depth_min"], kw["depth_max"], kw["voxel_size"], c2w[f]),
                              np_bounds(dcam, kw["depth_min"], kw["depth_max"], kw["voxel_size"], c2w[f]))
    o = FusionOracle(**kw)
    assert o.integrate(dcam, depth[:2], ccam, bgr[:2], c2w[:2], w2c[:2]) == 0
    vo = o.volume()
    coords, sdf, wt, col = np_fuse(s, kw, 2)
    k = _canon(coords)
    assert np.array_equal(vo["xyz"], coords[k].astype(np.int32))
    assert np.array_equal(vo["sdf"].view(np.uint32), sdf[k].view(np.uint32))
    assert np.array_equal(vo["weight"].view(np.uint32), wt[k].view(np.uint32))
    assert np.array_equal(vo["rgb"], col[k])
    assert (vo["weight"] > 0).sum() > 200


def test_kf2_synthetic_truth():
    """Fused sdf against the analytic signed distance of the bumpy sphere, for voxels within one voxel of the surface."""
    from intrinsic3d_b200.scene import _implicit
    import torch
    s = _scene(frames=6)
    kw = _okw(s)
    o = FusionOracle(**kw)
    assert o.integrate(*scene_inputs(s)) == 0
    o.finish(1)
    v = o.volume()
    vs = float(s["voxel_size"])
    truth = _implicit(torch.from_numpy(v["xyz"].astype(np.float64) * vs), torch.zeros(3, dtype=torch.float64), 10.0 * vs, 0.03).numpy()
    near = np.abs(truth) <= vs
    assert near.sum() > 500
    err = np.abs(v["sdf"][near] - truth[near])
    p95 = float(np.percentile(err, 95))
    print(f"KF2: {near.sum()} voxels within 1 voxel of the surface: |sdf - truth| mean {err.mean() / vs:.3f}, 95th percentile {p95 / vs:.3f}, "
          f"max {err.max() / vs:.3f} voxel")
    # projective distances overestimate at grazing angles (silhouettes): the tail is bounded by the truncation, the bulk is tight
    assert err.mean() <= 0.3 * vs and p95 <= 0.75 * vs and err.max() <= 5.0 * vs
    far = np.abs(truth) >= 2 * vs
    assert (np.sign(v["sdf"][far]) == np.sign(truth[far])).mean() >= 0.99


def test_kf3_correct_sdf_properties():
    """correctSDF's update flag is set by a double comparison against the float-stored value: float(dist_nb) can round above dist_nb,
    so the same update qualifies again every sweep and neither schedule stops before the cap on this scene.  What holds: no sign
    flips, magnitudes never grow, only weight > 0 survives clearing, and Jacobi and Gauss-Seidel agree on the voxel set, weights and
    colours; their sdf agree except in a few voxels (72 of 4612 here, by up to 0.96 voxel)."""
    s = _scene(frames=3)
    kw = _okw(s)
    o = FusionOracle(**kw)
    assert o.integrate(*scene_inputs(s)) == 0
    before = o.volume()
    g = o.clone()
    sj, sg = o.finish(1), g.finish(2)
    vj, vg = o.volume(), g.volume()
    for k in ("xyz", "weight", "rgb"):
        assert np.array_equal(vj[k], vg[k]), k
    diff = np.abs(vj["sdf"] - vg["sdf"])
    vs = np.float32(kw["voxel_size"])
    print(f"KF3: Jacobi {sj} sweeps, Gauss-Seidel {sg} sweeps; sdf differ in {(diff > 0).sum()} of {len(diff)} voxels, max {diff.max() / vs:.3f} voxel")
    assert (diff > 0).mean() <= 0.05 and diff.max() <= 1.0 * vs
    assert (vj["weight"] > 0).all()               # clearInvalidVoxels
    valid = before["weight"] > 0
    assert np.array_equal(vj["xyz"], before["xyz"][valid])
    assert ((vj["sdf"] >= 0) == (before["sdf"][valid] >= 0)).all()          # no sign flips
    assert (np.abs(vj["sdf"]) <= np.abs(before["sdf"][valid])).all()
    idx = {tuple(c): i for i, c in enumerate(vj["xyz"].tolist())}
    offs = np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3)
    worst = 0.0
    for i in np.random.default_rng(0).choice(len(vj["xyz"]), 1500, replace=False):
        c = vj["xyz"][i]
        sd = float(vj["sdf"][i])
        for off in offs:
            j = idx.get(tuple((c + off).tolist()))
            if j is None or j == i or (float(vj["sdf"][j]) >= 0) != (sd >= 0):
                continue
            dvec = c.astype(np.float32) * vs - (c + off).astype(np.float32) * vs
            dist = float(np.sqrt((dvec[0] * dvec[0] + dvec[1] * dvec[1]) + dvec[2] * dvec[2]))
            cand = float(vj["sdf"][j]) + (1.0 if sd >= 0 else -1.0) * dist
            worst = max(worst, abs(sd) - abs(cand))
    # after the 10-sweep cap the field is not at a fixed point on this scene (reported, not asserted)
    print(f"KF3: largest improvement a neighbour still offers after {sj} sweeps: {worst / vs:.4f} voxel")


def test_kf4_allocation_properties():
    s = _scene(frames=2)
    clip = (-0.02, 0.03, -0.05, 0.0, -0.05, 0.05)
    kw = _okw(s, clip=clip)
    dcam, depth, ccam, bgr, c2w, w2c = scene_inputs(s)
    o = FusionOracle(**kw)
    assert o.integrate(dcam, depth[:1], ccam, bgr[:1], c2w[:1], w2c[:1]) == 0
    v = o.volume()
    got = {tuple(c) for c in v["xyz"].tolist()}
    coords, *_ = np_fuse(s, kw, 1)
    assert got == {tuple(c) for c in coords.tolist()}
    # every voxel lies in the 27-block of some centre that passed the bounds and clip tests: the clipped box grown by one voxel
    vs = np.float32(kw["voxel_size"])
    w = v["xyz"].astype(np.float32) * vs
    assert (w[:, 0] >= np.float32(clip[0]) - vs * 1.01).all() and (w[:, 0] <= np.float32(clip[1]) + vs * 1.01).all()
    assert (w[:, 1] <= np.float32(clip[3]) + vs * 1.01).all()
    b = bounds(dcam, kw["depth_min"], kw["depth_max"], kw["voxel_size"], c2w[0])
    assert (v["xyz"][:, 0] >= b[0] - 1).all() and (v["xyz"][:, 0] <= b[1] + 1).all()


def test_kf4_first_sample_in_origin_voxel_is_skipped():
    """A single ray whose first sample falls into voxel (0,0,0) allocates nothing there: pos_grid_last starts at (0,0,0)."""
    vs = 0.004
    W, H = 3, 3
    cam = (W, H, 100.0, 100.0, 1.0, 1.0)
    depth = np.zeros((1, H, W), np.float32)
    depth[0, 1, 1] = 0.5                       # centre pixel: ray along +z
    bgr = np.zeros((1, H, W, 3), np.uint8)
    # camera at z = -(0.5 - 5 voxels): the first sample (d - trunc) lands exactly at the world origin
    c2w = np.array([[1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, -(0.5 - 5 * vs)]], np.float32)
    w2c = np.array([[1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, (0.5 - 5 * vs)]], np.float32)
    o = FusionOracle(voxel_size=vs, depth_min=0.1, depth_max=1.0, window=0)
    assert o.integrate(cam, depth, cam, bgr, c2w, w2c) == 0
    got = {tuple(c) for c in o.volume()["xyz"].tolist()}
    # the samples that fall into (0,0,0) are skipped, so the block of (0,0,-1) is never allocated; (0,0,1) onwards are centres
    assert (0, 0, 1) in got and (0, 0, 2) in got
    assert (0, 0, -1) not in got and (0, 0, -2) not in got
    assert (1, 1, 0) in got                    # (0,0,0) itself belongs to the block of (0,0,1)


def test_golden_fusion_fixture():
    g = np.load(os.path.join(HERE, "golden", "tiny_fusion.npz"))
    vs, dmin, dmax, ws = (float(x) for x in g["params"])
    o = FusionOracle(voxel_size=vs, depth_min=dmin, depth_max=dmax, weight_sample=ws, window=2, iterations=10)
    cam = tuple(g["cam"])
    assert o.integrate(cam, g["depth"], cam, g["bgr"], g["c2w"], g["w2c"]) == 0
    assert o.finish(1) == int(g["sweeps"])
    v = o.volume()
    for k in ("xyz", "sdf", "weight", "rgb"):
        assert np.array_equal(g[k], v[k]), k
