"""The bound of the conservative frame culling (frame_may_see and k_depth_tiles, i3d_observe.cuh / i3d_kernels.cuh), fuzzed on the
device by tests/native/check_cull.cu: for ~10^6 seeded (sphere, frame) cases with random cameras, strong lens distortion, principal
points outside the image, partial tiles, depth maps with NaN, +-inf, zero and negative pixels, and occlusion distances from "off" to
10 m, no case may be culled while a point of its sphere has a positive observation weight.  The spheres are placed where the bounds
are tight: on the occlusion band's edges, across the image borders, against the camera plane."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 32


def _lib():
    L = C.CDLL(os.path.join(ROOT, "tests", "native", "libcheck_cull.so"))
    L.check_cull.restype = C.c_int
    L.check_cull.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                             C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def run(depth, rt, cams, sph, frame, n_random=23, seed=1):
    """frame_may_see and the probed weights of every sphere; returns (may, hits, first hit point, (tile min, tile max))"""
    depth, rt, cams = (np.ascontiguousarray(a, np.float32) for a in (depth, rt, cams))
    sph, frame = np.ascontiguousarray(sph, np.float32), np.ascontiguousarray(frame, np.int32)
    F, H, W = depth.shape
    S = len(frame)
    TW, TH = -(-W // TILE), -(-H // TILE)
    may, hits = np.zeros(S, np.uint8), np.zeros(S, np.int32)
    pt, tiles = np.zeros((S, 3), np.float32), np.zeros((2, F, TH, TW), np.float32)
    rc = _lib().check_cull(F, W, H, depth.ctypes.data, rt.ctypes.data, cams.ctypes.data, S, sph.ctypes.data, frame.ctypes.data, n_random,
                           seed, may.ctypes.data, hits.ctypes.data, pt.ctypes.data, tiles.ctypes.data)
    assert rc == 0, f"CUDA error {rc}"
    return may.astype(bool), hits, pt, tiles


def tiles_ref(depth):
    """per 32x32 tile: the least positive depth (+inf if none) and the largest, +inf if the tile has a NaN pixel"""
    F, H, W = depth.shape
    TW, TH = -(-W // TILE), -(-H // TILE)
    pad = np.full((F, TH * TILE, TW * TILE), -1.0, np.float32)
    pad[:, :H, :W] = depth
    t = pad.reshape(F, TH, TILE, TW, TILE).transpose(0, 1, 3, 2, 4).reshape(F, TH, TW, TILE * TILE)
    pos = t > 0
    tmin = np.where(pos, t, np.inf).min(-1).astype(np.float32)
    tmax = np.where(pos, t, 0.0).max(-1).astype(np.float32)
    tmax[np.isnan(t).any(-1)] = np.inf
    return tmin, tmax


def _rotation(rng, n):
    w = rng.standard_normal((n, 3)) * rng.uniform(0, np.pi, (n, 1)) / np.sqrt(3)
    th = np.linalg.norm(w, axis=1)[:, None, None]
    k = w / np.maximum(np.linalg.norm(w, axis=1, keepdims=True), 1e-12)
    Kx = np.zeros((n, 3, 3))
    Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    Kx[:, 1, 0], Kx[:, 2, 0], Kx[:, 2, 1] = k[:, 2], -k[:, 1], k[:, 0]
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


DISTORTIONS = [np.zeros(5), np.array([0.03, -0.01, 0.004, 0.002, -0.0015]), np.array([-0.4, 0.12, -0.02, 0.01, -0.01]),
               np.array([0.3, -0.08, 0.02, -0.01, 0.01]), np.array([-0.4, 0.0, 0.0, 0.01, 0.01])]
OCCLUSIONS = [0.0, -1.0, 1e-6, 0.02, 10.0]


def world(rng, F, W, H):
    """F frames of W x H: cameras, distortion (d = k1, k2, k3, p1, p2), occlusion distance and a depth map with every hazard"""
    R = _rotation(rng, F)
    C_ = rng.uniform(-1, 1, (F, 3))
    rt = np.zeros((F, 12))
    rt[:, :9] = R.reshape(F, 9)
    rt[:, 9:] = -np.einsum("fij,fj->fi", R, C_)
    cams = np.zeros((F, 10))
    fx = W * rng.uniform(0.3, 3.0, F)
    cams[:, 0], cams[:, 1] = fx, fx * rng.uniform(0.8, 1.25, F)
    off = rng.random(F) < 0.25                               # principal point far off-centre, or outside the image
    cams[:, 2] = np.where(off, rng.uniform(-0.5, 1.5, F) * W, (W - 1) * 0.5 + rng.uniform(-3, 3, F))
    cams[:, 3] = np.where(off, rng.uniform(-0.5, 1.5, F) * H, (H - 1) * 0.5 + rng.uniform(-3, 3, F))
    cams[:, 4:9] = np.array(DISTORTIONS)[rng.integers(0, len(DISTORTIONS), F)]
    cams[:, 9] = np.array(OCCLUSIONS)[np.arange(F) % len(OCCLUSIONS)]
    # depth: constant over 8x8 blocks (tight tile bounds), then per frame one hazard
    blk = rng.uniform(0.2, 4.0, (F, -(-H // 8), -(-W // 8))).astype(np.float32)
    depth = np.repeat(np.repeat(blk, 8, 1), 8, 2)[:, :H, :W].copy()
    for f in range(F):
        hz = f % 8
        if hz == 1:
            depth[f] = np.nan                                                    # a dropped frame
        elif hz == 2:                                                            # NaN 32x32 blocks
            for _ in range(3):
                y, x = rng.integers(0, max(1, H - 8)), rng.integers(0, max(1, W - 8))
                depth[f, y:y + 32, x:x + 32] = np.nan
        elif hz == 3:
            depth[f][rng.random((H, W)) < 0.05] = np.nan                          # scattered NaN pixels
        elif hz == 4:                                                            # NaN mixed with 0
            m = rng.random((H, W)) < 0.5
            depth[f] = np.where(m, np.nan, 0.0)
        elif hz == 5:
            r = rng.random((H, W))
            depth[f][r < 0.03] = np.inf
            depth[f][(r >= 0.03) & (r < 0.06)] = -np.inf
            depth[f][(r >= 0.06) & (r < 0.1)] = np.nan
        elif hz == 6:
            depth[f][rng.random((H, W)) < 0.3] = 0.0
            depth[f][rng.random((H, W)) < 0.1] = -1.0
    # a few non-finite poses
    if F >= 8:
        rt[3, 11] = np.nan
        rt[5, 9] = np.inf
        rt[7, 0] = np.inf
    return rt, cams, depth


def spheres(rng, rt, cams, depth, S):
    """S spheres, each aimed at a frame: centre near a pixel in and around the image at a depth on the edge of the occlusion band of the
    depth under it, at a random depth, or against the camera plane; footprints from a fraction of a pixel to a few tiles"""
    F, H, W = depth.shape
    f = rng.integers(0, F, S)
    fx, fy, cx, cy, occ = cams[f, 0], cams[f, 1], cams[f, 2], cams[f, 3], cams[f, 9]
    u = rng.uniform(-0.25, 1.25, S) * W
    v = rng.uniform(-0.25, 1.25, S) * H
    iu, iv = np.clip(u.astype(int), 0, W - 1), np.clip(v.astype(int), 0, H - 1)
    dref = depth[f, iv, iu].astype(np.float64)
    dref = np.where(np.isfinite(dref) & (dref > 0), dref, rng.uniform(0.2, 4.0, S))
    rpx = np.exp(rng.uniform(np.log(0.05), np.log(120.0), S))
    mode = rng.integers(0, 4, S)
    z = np.where(mode == 0, dref * rng.uniform(0.5, 1.5, S), dref)
    rad = z * rpx / fx
    # occlusion edges: nearest or farthest point of the sphere at d -+ occ (relative offsets down to 1e-7)
    sgn = np.where(rng.random(S) < 0.5, -1.0, 1.0)
    eps = rng.choice([-1e-3, -1e-5, -1e-7, 0.0, 1e-7, 1e-5, 1e-3], S)
    edge = dref + sgn * (np.maximum(occ, 0) + rad) * (1 + eps)
    z = np.where(mode >= 2, edge, z)
    # against the camera plane: zmin around 1e-3
    near = rng.random(S) < 0.08
    rad = np.where(near, rng.uniform(1e-4, 0.05, S), rad)
    z = np.where(near, rad + rng.uniform(-2e-3, 5e-3, S), z)
    x, y = (u - cx) / fx * z, (v - cy) / fy * z
    q = np.stack([x, y, z], 1)
    Rm = rt[f, :9].reshape(S, 3, 3)
    Rm = np.where(np.isfinite(Rm), Rm, 0.0)
    t = np.where(np.isfinite(rt[f, 9:]), rt[f, 9:], 0.0)
    c = np.einsum("sji,sj->si", Rm, q - t)
    return np.concatenate([c, rad[:, None]], 1), f


def test_depth_tiles_rule():
    """k_depth_tiles against its rule at partial tiles, with NaN, +-inf, zero and negative pixels"""
    rng = np.random.default_rng(3)
    for W, H in ((33, 31), (100, 75), (64, 48)):
        rt, cams, depth = world(rng, 16, W, H)
        _, _, _, tiles = run(depth, rt, cams, np.zeros((1, 4)), np.zeros(1))
        tmin, tmax = tiles_ref(depth)
        assert tiles[0].tobytes() == tmin.tobytes() and tiles[1].tobytes() == tmax.tobytes(), (W, H)


@pytest.mark.parametrize("occlusion", [0.0, -1.0])
def test_nan_depth_is_observed_without_occlusion_test(occlusion):
    """With the occlusion test off the reference observes a NaN depth (it rejects d <= 0 only): a frame that is NaN under the sphere, in
    whole or in part, must not be culled"""
    W, H = 100, 75
    depth = np.full((4, H, W), np.nan, np.float32)
    depth[1, :, 50:] = 0.0                                          # NaN mixed with 0
    depth[2, ::2, ::2] = 0.0
    depth[3] = 0.0                                                  # NaN in one 32x32 block
    depth[3, 32:64, 32:64] = np.nan
    rt = np.zeros((4, 12))
    rt[:, [0, 4, 8]] = 1.0
    cams = np.tile([80.0, 80.0, 49.5, 37.0, 0, 0, 0, 0, 0, occlusion], (4, 1))
    sph = np.array([[0.0, 0.0, 1.0, 0.01], [0.1, 0.05, 0.8, 0.003], [-0.2, 0.1, 1.5, 0.02], [0.0, 0.0, 1.0, 0.005]])
    frame = np.tile(np.arange(4), 4)
    may, hits, _, _ = run(depth, rt, cams, np.repeat(sph, 4, 0), frame)
    assert set(frame[hits > 0]) == {0, 1, 2, 3}
    assert may[hits > 0].all(), np.nonzero(~may & (hits > 0))[0]
    # with the occlusion test on, NaN is rejected, and the culling still drops the all-NaN frame
    cams[:, 9] = 0.02
    may, hits, _, _ = run(depth, rt, cams, sph[:1], [0])
    assert hits[0] == 0 and not may[0]


@pytest.mark.parametrize("W,H", [(33, 31), (100, 75), (64, 48), (160, 120)])
def test_cull_bound_fuzz(W, H):
    """~2.6 * 10^5 spheres per size: a culled (sphere, frame) pair never has a probed point of positive weight, and the culling drops a
    fair share of the pairs, so the claim is tested where it acts"""
    rng = np.random.default_rng(W * 1000 + H)
    S, F = 1 << 18, 64
    rt, cams, depth = world(rng, F, W, H)
    sph, frame = spheres(rng, rt, cams, depth, S)
    may, hits, pt, _ = run(depth, rt, cams, sph, frame, seed=W * H)
    bad = np.nonzero(~may & (hits > 0))[0]
    culled = int((~may).sum())
    seen = int((hits > 0).sum())
    print(f"cull bound {W}x{H}: {S} spheres, {culled} culled ({100.0 * culled / S:.1f} %), {seen} with a visible probe, "
          f"{len(bad)} culled but visible")
    assert len(bad) == 0, [(int(i), int(frame[i]), sph[i].tolist(), pt[i].tolist(), cams[frame[i]].tolist()) for i in bad[:5]]
    assert culled >= 0.2 * S and seen >= 0.1 * S
