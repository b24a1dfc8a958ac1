"""CPU tests of the surface-distance restatement tests/distance_ref.py (DESIGN.md §6u): the closest point on a triangle against float64,
the samples, known answers, the indexed query against brute force, the truth mesh's own error and the fixture."""
import os

import numpy as np
import pytest

import distance_ref as dr

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32


def _seg64(p, a, b):
    e = b - a
    ll = (e * e).sum(-1)
    t = np.clip(np.where(ll > 0, ((p - a) * e).sum(-1) / np.where(ll > 0, ll, 1.0), 0.0), 0.0, 1.0)
    q = a + t[:, None] * e
    return ((p - q) ** 2).sum(-1), t


def _tri64(p, a, b, c):
    """float64 d^2 and the part of the triangle that is closest: 0 interior, 1 + k edge k (ab, bc, ca), 4 + k vertex k"""
    n = np.cross(b - a, c - a)
    nn = (n * n).sum(-1)
    ok = nn > 0
    s = np.where(ok, ((p - a) * n).sum(-1) / np.where(ok, nn, 1.0), 0.0)
    q = p - s[:, None] * n
    # barycentric of the projection
    v0, v1, v2 = b - a, c - a, q - a
    d00, d01, d11, d20, d21 = (v0 * v0).sum(-1), (v0 * v1).sum(-1), (v1 * v1).sum(-1), (v2 * v0).sum(-1), (v2 * v1).sum(-1)
    den = np.where(ok, d00 * d11 - d01 * d01, 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        v = (d11 * d20 - d01 * d21) / den
        w = (d00 * d21 - d01 * d20) / den
        inside = ok & (nn > 1e-9 * (v0 * v0).sum(-1) * (v1 * v1).sum(-1)) & (v >= 0) & (w >= 0) & (v + w <= 1)
    segs = [_seg64(p, a, b), _seg64(p, b, c), _seg64(p, c, a)]
    ds = np.stack([d for d, _ in segs])
    k = np.argmin(ds, 0)
    d2 = np.where(inside, ((p - q) ** 2).sum(-1), ds.min(0))
    t = np.stack([t for _, t in segs])[k, np.arange(len(p))]
    part = np.where(inside, 0, np.where(t <= 0, 4 + k, np.where(t >= 1, 4 + (k + 1) % 3, 1 + k)))
    return d2, part


def _random_case(rng, n, degenerate=None):
    a, b, c = (rng.normal(0, 1, (n, 3)) for _ in range(3))
    if degenerate == "collinear":
        c = a + rng.uniform(-1, 2, (n, 1)) * (b - a)
    elif degenerate == "point":
        b = a.copy()
        c = a.copy()
    elif degenerate == "edge":
        b = a.copy()
    p = rng.normal(0, 1.5, (n, 3))
    return [x.astype(f32) for x in (p, a, b, c)]


@pytest.mark.parametrize("degenerate", [None, "collinear", "point", "edge"])
def test_point_triangle_against_float64(degenerate):
    rng = np.random.default_rng(3)
    p, a, b, c = _random_case(rng, 20000, degenerate)
    d2 = dr.point_tri_d2(p, a, b, c)
    ref, part = _tri64(*(x.astype(np.float64) for x in (p, a, b, c)))
    scale = 1.0 + np.abs(np.stack([p, a, b, c])).max(axis=(0, 2)).astype(np.float64) ** 2
    err = np.abs(d2.astype(np.float64) - ref) / scale
    assert err.max() < 2e-5, err.max()
    if degenerate is None:
        assert set(np.unique(part)) == set(range(7))         # interior, the three edges and the three vertices are each hit


def test_point_triangle_against_dense_sampling():
    rng = np.random.default_rng(4)
    p, a, b, c = _random_case(rng, 200)
    n = 120
    u, v = np.meshgrid(np.arange(n + 1) / n, np.arange(n + 1) / n)
    k = (u + v) <= 1
    u, v = u[k], v[k]
    pts = a.astype(np.float64)[:, None] + u[None, :, None] * (b - a)[:, None] + v[None, :, None] * (c - a)[:, None]
    dense = ((pts - p[:, None].astype(np.float64)) ** 2).sum(-1).min(1)
    d2 = dr.point_tri_d2(p, a, b, c).astype(np.float64)
    assert np.all(d2 <= dense * (1 + 1e-5) + 1e-6)                     # never above a point of the triangle
    edge = np.linalg.norm(np.stack([b - a, c - b, a - c]), axis=2).max(0)
    assert np.all(np.sqrt(dense) - np.sqrt(d2) <= edge / n + 1e-5)       # and within the sampling step of its minimum


@pytest.mark.parametrize("L", [1, 2, 3, 5, 16])
def test_samples(L):
    rng = np.random.default_rng(L)
    mesh = dict(vertices=rng.normal(0, 1, (30, 3)).astype(f32), faces=rng.integers(0, 30, (40, 3)).astype(np.int32))
    mesh["faces"][0] = [1, 1, 2]                                        # a zero-area face
    P, w = dr.samples(mesh, L)
    assert P.shape == (40 * L * L, 3) and w.shape == (40 * L * L,)
    area = dr.face_area(mesh["vertices"], mesh["faces"]).astype(np.float64)
    np.testing.assert_allclose(w.reshape(40, -1).sum(1), area, rtol=1e-14)
    assert np.all(w[: L * L] == 0)
    a, b = dr.sample_bary(L)
    assert len(a) == L * L and np.all(a > 0) and np.all(b > 0) and np.all(a + b < 1)
    # the centroids of the L^2 congruent sub-triangles, each sub-triangle once
    up = [((i + 1 / 3) / L, (j + 1 / 3) / L) for i in range(L) for j in range(L - i)]
    down = [((i + 2 / 3) / L, (j + 2 / 3) / L) for i in range(L - 1) for j in range(L - 1 - i)]
    np.testing.assert_allclose(np.stack([a, b], 1), np.array(up + down), atol=1e-6)
    assert len(set(up + down)) == L * L
    # every sample on its face (barycentric reconstruction in float64)
    v = mesh["vertices"].astype(np.float64)
    f = mesh["faces"]
    q = (1 - a - b)[None, :, None] * v[f[:, 0]][:, None] + a[None, :, None] * v[f[:, 1]][:, None] + b[None, :, None] * v[f[:, 2]][:, None]
    np.testing.assert_allclose(P.reshape(40, L * L, 3), q, atol=1e-5)


def _square(z, n=4):
    x = np.arange(n + 1, dtype=f32) / f32(n)
    X, Y = np.meshgrid(x, x, indexing="ij")
    v = np.stack([X.ravel(), Y.ravel(), np.full(X.size, f32(z))], 1).astype(f32)
    i = (np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]).ravel()
    f = np.concatenate([np.stack([i, i + n + 1, i + n + 2], 1), np.stack([i, i + n + 2, i + 1], 1)])
    return dict(vertices=v, faces=f.astype(np.int32))


def test_parallel_squares():
    h = 0.25
    a, b = _square(0.0), _square(h)
    r = dr.distance(a, b, 3, 1.0, [0.5 * h, 0.999 * h, 1.001 * h, 2 * h])
    for side in ("accuracy", "completeness"):
        assert r[side]["num_matched"] == r[side]["num_samples"]
        np.testing.assert_allclose(np.sqrt(r[side + "_d2"].astype(np.float64)), h, rtol=1e-6)
        assert r[side]["fraction"] == [0.0, 0.0, 1.0, 1.0]
    assert r["precision"] == r["recall"] == r["fscore"] == [0.0, 0.0, 1.0, 1.0]
    np.testing.assert_allclose(r["vertex_distance"], h, rtol=1e-6)


def _sphere(n_theta=24, r=0.1):
    from intrinsic3d_b200.scene import _latlong
    d, f = _latlong(n_theta)
    return dict(vertices=(r * d).astype(f32), faces=f.astype(np.int32))


def test_hemisphere_against_sphere_and_self():
    s = _sphere()
    v = s["vertices"]
    cz = v[s["faces"]].mean(1)[:, 2]
    hemi = dict(vertices=v, faces=s["faces"][cz > 0])
    tau = [0.001, 0.005]
    r = dr.distance(hemi, s, 2, 0.05, tau)
    assert r["precision"] == [1.0, 1.0]
    assert r["accuracy"]["max"] < 1e-6
    assert abs(r["recall"][0] - 0.5) < 0.02 and r["recall"][0] < 1
    # the sphere's lower samples lie outside the hemisphere's box: matched only within max_distance
    assert r["completeness"]["num_matched"] < r["completeness"]["num_samples"] or r["completeness"]["max"] > 0.01
    # a mesh against itself: every distance within float rounding
    r = dr.distance(s, s, 3, 0.05, tau)
    for side in ("accuracy", "completeness"):
        assert np.sqrt(r[side + "_d2"].max()) < 1e-6 and r[side]["num_matched"] == r[side]["num_samples"]
    assert r["fscore"] == [1.0, 1.0] and np.all(r["vertex_distance"] == 0)


def test_tie_goes_to_lowest_face():
    v = np.array([[-1, -1, -1], [1, -1, -1], [0, 1, -1], [-1, -1, 1], [1, -1, 1], [0, 1, 1], [5, 5, 5], [6, 5, 5], [5, 6, 5]], f32)
    P = np.array([[0, 0, 0], [0.1, -0.2, 0]], f32)
    for faces, want in (([[6, 7, 8], [0, 1, 2], [3, 4, 5]], 1), ([[3, 4, 5], [0, 1, 2], [6, 7, 8]], 0), ([[0, 1, 2], [3, 4, 5]], 0)):
        m = dict(vertices=v, faces=np.array(faces, np.int32))
        for q in (dr.nearest, dr.nearest_brute):
            d2, f = q(P, m, 2.0)
            assert np.all(d2 == 1.0) and np.all(f == want), (faces, q, d2, f)


def test_indexed_query_equals_brute_force():
    from intrinsic3d_b200.scene import config_geometry, truth_mesh
    rng = np.random.default_rng(9)
    m = truth_mesh(16, **config_geometry("tiny"))
    P, _ = dr.samples(m, 2)
    P = np.concatenate([P + rng.normal(0, 0.003, P.shape).astype(f32), rng.uniform(-0.08, 0.08, (500, 3)).astype(f32)])
    for maxd in (0.002, 0.01, 1.0):
        a, b = dr.nearest_brute(P, m, maxd), dr.nearest(P, m, maxd)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), maxd
        assert (a[1] < 0).any() == (maxd < 1.0)


@pytest.mark.parametrize("name", ["tiny", "small", "c2", "c3"])
def test_truth_mesh_error(name):
    from intrinsic3d_b200.scene import config_geometry, truth_mesh, truth_mesh_error
    g = config_geometry(name)
    m = truth_mesh(**g)
    err = truth_mesh_error(m, **g)
    vs = g["voxel_size"]
    assert err < 0.01 * vs, (name, err)          # measured: 0.29 %, 0.58 %, 0.15 % and 0.075 % of a voxel
    assert m["faces"].min() == 0 and m["faces"].max() == len(m["vertices"]) - 1
    if name == "c3":
        assert 2e6 < len(m["faces"]) < 8e6


def test_golden_fixture():
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden_distance as mg
    g = np.load(os.path.join(HERE, "golden", "tiny_distance.npz"))
    m, t, maxd, taus = mg.inputs()
    assert m["faces"].tobytes() == g["faces"].tobytes() and t["faces"].tobytes() == g["truth_faces"].tobytes()
    r = dr.distance(m, t, int(g["L"]), maxd, taus)
    for k in ("accuracy_d2", "accuracy_face", "completeness_d2", "completeness_face", "vertex_distance", "vertex_face"):
        assert r[k].tobytes() == g[k].tobytes(), k
    d2, f = dr.nearest_brute(dr.samples(m, int(g["L"]))[0], t, maxd)
    assert d2.tobytes() == g["accuracy_d2"].tobytes() and f.tobytes() == g["accuracy_face"].tobytes()
