"""CPU tests of the texture bake's restatement (tests/texture_ref.py, DESIGN.md §6t): the atlas layout and its no-bleed property, the
texel-to-point map, known answers, the PNG and OBJ writers, the fixture, and the measured gain of the texture over the vertex colours."""
import os
import struct
import zlib

import numpy as np
import pytest

import texture_ref as tr

f32 = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))


def _taps(u, v):
    """The four texels of a bilinear lookup at local (u, v) (texel centres at half-integers) and their weights."""
    i0, j0 = np.floor(u - 0.5).astype(np.int64), np.floor(v - 0.5).astype(np.int64)
    fu, fv = (u - 0.5) - i0, (v - 0.5) - j0
    return [(i0 + di, j0 + dj, (fu if di else 1 - fu) * (fv if dj else 1 - fv)) for di in (0, 1) for dj in (0, 1)]


@pytest.mark.parametrize("S", [6, 7, 8, 12, 33, 256])
def test_bilinear_lookup_reads_only_owned_texels(S):
    rng = np.random.default_rng(S)
    for face_b in (False, True):
        c = tr.uv_corners(S, face_b).astype(np.float64)
        r = rng.random((20000, 2))
        r = np.where(r.sum(1, keepdims=True) > 1, 1 - r, r)             # uniform in the triangle
        pts = c[0] + r[:, :1] * (c[1] - c[0]) + r[:, 1:] * (c[2] - c[0])
        # and the corners, edge midpoints and points along each edge, where some taps have weight 0
        t = np.linspace(0, 1, 41)[:, None]
        edges = np.concatenate([c[a] + t * (c[b] - c[a]) for a, b in ((0, 1), (1, 2), (2, 0))])
        for P, need_all in ((pts, True), (edges, False)):
            for i, j, w in _taps(P[:, 0], P[:, 1]):
                live = np.ones(len(P), bool) if need_all else w > 0
                assert np.all((i[live] >= 0) & (i[live] < S) & (j[live] >= 0) & (j[live] < S)), (S, face_b)
                assert np.all(tr.owns(S, face_b, i[live], j[live])), (S, face_b)
        # the owned sets of A and B are disjoint, and each has S (S - 1) / 2 texels
        i, j = np.meshgrid(np.arange(S), np.arange(S))
        assert not np.any(tr.owns(S, False, i, j) & tr.owns(S, True, i, j))
        assert tr.owns(S, face_b, i, j).sum() == S * (S - 1) // 2


@pytest.mark.parametrize("F", [1, 2, 3, 7, 8, 51])
def test_layout_and_owned_texels(F):
    S = 8
    L = tr.layout(F, S)
    ncells = (F + 1) // 2
    assert L["cols"] ** 2 >= ncells and (L["cols"] - 1) ** 2 < ncells and L["rows"] * L["cols"] >= ncells
    face, i, j, x, y = tr.owned_texels(F, S)
    assert len(face) == F * S * (S - 1) // 2
    assert len(set(zip(x.tolist(), y.tolist()))) == len(face)                  # every atlas texel belongs to at most one face
    assert np.all((x // S) + L["cols"] * (y // S) == face // 2)                 # inside its own cell
    # kernel order: cell-major, row-major inside a cell
    key = (face // 2) * S * S + j * S + i
    assert np.all(np.diff(key) > 0)


def test_uv_corners_map_to_vertices_and_points_lie_on_the_face():
    rng = np.random.default_rng(1)
    for S in (6, 12, 40):
        for face_b in (False, True):
            c = tr.uv_corners(S, face_b)
            for scale in (1e-3, 1.0, 7.0):
                p = (rng.standard_normal((500, 3, 3)) * scale + rng.standard_normal((500, 1, 3))).astype(f32)
                for k in range(3):
                    a, b = tr.bary(S, np.full(500, face_b), np.full(500, c[k, 0]), np.full(500, c[k, 1]))
                    P, _ = tr.point(a, b, p[:, 0], p[:, 1], p[:, 2])
                    assert np.array_equal(P, p[:, k]), (S, face_b, k)
    # every texel point lies on its face's plane, to float32 rounding
    p = rng.standard_normal((300, 3)).astype(f32)
    faces = rng.choice(300, (400, 3), replace=True)
    faces = faces[(faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])]
    mesh = dict(vertices=p, faces=faces, colors=np.zeros((300, 3), np.uint8))
    tp = tr.texel_points(mesh, 12)
    p0 = p[faces[tp["face"], 0]].astype(np.float64)
    n = np.cross(p[faces[:, 1]].astype(np.float64) - p[faces[:, 0]], p[faces[:, 2]].astype(np.float64) - p[faces[:, 0]])
    n = n / np.linalg.norm(n, axis=1, keepdims=True)
    dist = np.abs(((tp["P"].astype(np.float64) - p0) * n[tp["face"]]).sum(1))
    assert dist.max() <= 1e-5, dist.max()
    assert np.all(tp["a"] >= 0) and np.all(tp["b"] >= 0) and np.all(tp["a"] + tp["b"] <= 1 + 1e-6)


def _flat_square(z=1.0, half=0.3, n=4):
    """A flat square at depth z, facing the camera at the origin: an n x n grid of vertices, 2 (n-1)^2 faces."""
    g = np.linspace(-half, half, n)
    X, Y = np.meshgrid(g, g)
    v = np.stack([X.ravel(), Y.ravel(), np.full(n * n, z)], 1).astype(f32)
    f = []
    for r in range(n - 1):
        for c in range(n - 1):
            a, b, d, e = r * n + c, r * n + c + 1, (r + 1) * n + c, (r + 1) * n + c + 1
            f += [[a, b, d], [b, e, d]]
    return v, np.array(f, np.int32)


def _camera(W=96, H=80, fx=90.0):
    import render_ref as rr
    return rr.camera([fx, fx, (W - 1) / 2, (H - 1) / 2], np.zeros(5)), W, H


def test_known_answer_fronto_parallel_square():
    cam, W, H = _camera()
    v, f = _flat_square()
    rng = np.random.default_rng(2)
    img = rng.integers(0, 256, (1, H, W, 3), dtype=np.uint8)
    depth = np.ones((1, H, W), f32)
    rt = np.array([[1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]], f32)
    mesh = dict(vertices=v, faces=f, colors=np.zeros((len(v), 3), np.uint8))
    for K in (0, 1, 5):
        b = tr.bake(mesh, depth, img, rt, cam, 12, 0.02, K)
        assert b["info"]["num_texels_fallback"] == 0 and b["info"]["num_observations"] == b["info"]["num_texels_owned"]
        tp = tr.texel_points(mesh, 12)
        P = tp["P"].astype(np.float64)
        pu, pv = cam["fx"] * P[:, 0] / P[:, 2] + cam["cx"], cam["fy"] * P[:, 1] / P[:, 2] + cam["cy"]
        got = b["image"][tp["y"], tp["x"]].astype(int)
        for k, ch in enumerate((2, 1, 0)):
            want = tr.interp_u8(img[0], pu.astype(f32), pv.astype(f32), ch).astype(int)
            # one observation: c (w / 255) (255 / w) truncates to c or c - 1, and the projection here is float64, so a bilinear value
            # on a truncation boundary may land one above
            d = want - got[:, k]
            assert np.abs(d).max() <= 1 and (d == 0).mean() > 0.95, np.unique(d, return_counts=True)


def test_known_answer_constant_frames_and_unseen_faces():
    cam, W, H = _camera()
    v, f = _flat_square()
    vcol = np.random.default_rng(3).integers(0, 256, (len(v), 3), dtype=np.uint8)
    mesh = dict(vertices=v, faces=f, colors=vcol)
    img = np.empty((3, H, W, 3), np.uint8)
    img[...] = np.array([40, 120, 200], np.uint8)                      # B, G, R
    depth = np.ones((3, H, W), f32)
    rt = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], f32), (3, 1))
    rt[1, 9], rt[2, 10] = 0.01, -0.02
    b = tr.bake(mesh, depth, img, rt, cam, 8, 0.05, 5)
    tp = tr.texel_points(mesh, 8)
    got = b["image"][tp["y"], tp["x"]].astype(int)
    assert np.all(np.abs(got - np.array([200, 120, 40])) <= 1)
    # no frame sees the square (the depth is 0.5 m in front of it): every texel is the barycentric blend of the vertex colours
    b = tr.bake(mesh, depth * f32(0.5), img, rt, cam, 8, 0.05, 5)
    assert b["info"]["num_texels_observed"] == 0 and b["info"]["num_texels_fallback"] == b["info"]["num_texels_owned"]
    fv = f[tp["face"]]
    want = sum(wk[:, None] * vcol[fv[:, q]].astype(np.float64) for q, wk in enumerate((tp["w0"], tp["a"], tp["b"])))
    got = b["image"][tp["y"], tp["x"]].astype(int)
    assert np.abs(got - np.floor(want + 0.5)).max() <= 1
    # constant vertex colours give that constant exactly
    mesh1 = dict(vertices=v, faces=f, colors=np.tile(np.array([[9, 130, 254]], np.uint8), (len(v), 1)))
    b = tr.bake(mesh1, depth * f32(0.5), img, rt, cam, 8, 0.05, 5)
    assert np.all(b["image"][tp["y"], tp["x"]] == np.array([9, 130, 254]))
    # the unused texels hold 0
    used = np.zeros(b["image"].shape[:2], bool)
    used[tp["y"], tp["x"]] = True
    assert not b["image"][~used].any()


def _tiny_inputs():
    import mesh_ref
    import render_ref as rr
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = config_scene("tiny")
    col = make_color_frames(s)
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], s["rgb"], float(s["voxel_size"]), True)
    return s, col, m, rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"])


def test_k_handling():
    """As the recolouring's KR2: the counts do not depend on K; K above the number of frames is K = 0; K = 1 changes the texels with more
    than one observation."""
    s, col, m, rt, cam = _tiny_inputs()
    b = {K: tr.bake(m, s["depth"], col, rt, cam, 8, 0.02, K) for K in (0, 1, 5, 8)}
    for K in (1, 5, 8):
        for k in ("num_texels_observed", "num_observations", "num_texels_fallback"):
            assert b[K]["info"][k] == b[0]["info"][k]
    assert len(rt) < 8 and b[8]["image"].tobytes() == b[0]["image"].tobytes()
    assert b[1]["info"]["num_observations_kept"] == b[1]["info"]["num_texels_observed"]
    assert b[1]["info"]["num_observations"] > 1.5 * b[1]["info"]["num_texels_observed"]
    assert (b[1]["image"] != b[0]["image"]).any(2).sum() > 0.3 * b[0]["info"]["num_texels_observed"]


def _png_decode(data):
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, hdr = 8, b"", None
    while pos < len(data):
        n, tag = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(tag + body) & 0xFFFFFFFF
        if tag == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"IDAT":
            idat += body
        pos += 12 + n
    W, H, depth, ctype, _, _, _ = hdr
    assert depth == 8 and ctype == 2
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(H, 1 + 3 * W)
    assert not raw[:, 0].any()                                          # filter 0 on every scanline
    return raw[:, 1:].reshape(H, W, 3)


def test_png_and_obj_round_trip(tmp_path):
    from intrinsic3d_b200.mesh import obj_bytes, png_bytes, save_textured_obj
    s, col, m, rt, cam = _tiny_inputs()
    b = tr.bake(m, s["depth"], col, rt, cam, 6, 0.02, 5)
    data = png_bytes(b["image"])
    assert data == png_bytes(b["image"].copy())
    assert _png_decode(data).tobytes() == b["image"].tobytes()
    paths = save_textured_obj(str(tmp_path / "t"), m, b)
    assert open(paths[0], "rb").read() == obj_bytes(m, b["uv"], "t.mtl")
    assert "map_Kd t.png" in open(paths[1]).read()
    assert _png_decode(open(paths[2], "rb").read()).tobytes() == b["image"].tobytes()
    v, vt, faces = [], [], []
    for line in open(paths[0]).read().splitlines():
        tok = line.split()
        if tok[0] == "v":
            v.append([f32(float(x)) for x in tok[1:]])
        elif tok[0] == "vt":
            vt.append([f32(float(x)) for x in tok[1:]])
        elif tok[0] == "f":
            faces.append([[int(p) - 1 for p in x.split("/")] for x in tok[1:]])
    faces = np.array(faces)
    assert np.array(v, f32).tobytes() == m["vertices"].tobytes()
    assert np.array(vt, f32).tobytes() == b["uv"].reshape(-1, 2).tobytes()
    assert np.array_equal(faces[:, :, 0], m["faces"]) and np.array_equal(faces[:, :, 1], np.arange(3 * len(faces)).reshape(-1, 3))
    with pytest.raises(ValueError):
        png_bytes(np.zeros((0, 4, 3), np.uint8))


def _truth(s, P, radius_vox):
    """The scene's analytic albedo * shading at the surface point radially closest to P."""
    import torch
    from intrinsic3d_b200 import scene as sc
    vs = float(np.float32(s["voxel_size"]))
    rho0, bump = radius_vox * vs, 0.03
    p = torch.tensor(P, dtype=torch.float64)
    d = p / torch.linalg.norm(p, dim=-1, keepdim=True)
    ps = d * sc._rho(d, rho0, bump)[..., None]
    n = sc._normal(ps, torch.zeros(3, dtype=torch.float64), rho0, bump)
    a = sc._albedo_truth(ps, max(6.0 * vs, rho0 / 4.0))
    return (a * (sc.sh_basis(n) * torch.tensor(s["sh"][0])).sum(-1)).numpy()


# Mean absolute intensity error against the analytic appearance after recompute_colors (K = 5) and simplification at 4 voxels, S = 12,
# over every owned texel: (texture, barycentric vertex colours).  Measured: tiny 0.0548 / 0.1055, small 0.0492 / 0.1198.
QUALITY_BOUND = 0.065


@pytest.mark.parametrize("name,radius_vox", [("tiny", 10.0), ("small", 20.0)])
def test_texture_beats_vertex_colours(name, radius_vox):
    import mesh_ref
    import mesh_simplify_ref as msr
    import oracle
    import render_ref as rr
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = config_scene(name)
    col = make_color_frames(s)
    o = oracle.Oracle(threads=4)
    o.load_scene(s)
    o.set_color_frames(col)
    o.recompute_colors(0.02, 5)
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], o.colors(), float(s["voxel_size"]), False)
    m = msr.simplify(m, 4 * float(s["voxel_size"]))
    b = tr.bake(m, s["depth"], col, rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"]), 12, 0.02, 5)
    tp = tr.texel_points(m, 12)
    truth = _truth(s, tp["P"].astype(np.float64), radius_vox)
    gain = 255.0 * (1.0 + 0.92 + 0.85)                                 # make_color_frames' mean channel gains
    tex = b["image"][tp["y"], tp["x"]].astype(np.float64).sum(1) / gain
    fv = m["faces"][tp["face"]]
    vc = m["colors"].astype(np.float64)
    vert = sum(w[:, None].astype(np.float64) * vc[fv[:, q]] for q, w in enumerate((tp["w0"], tp["a"], tp["b"]))).sum(1) / gain
    e_tex, e_vert = np.abs(tex - truth).mean(), np.abs(vert - truth).mean()
    print(name, len(m["faces"]), "texture MAE %.4f, vertex colours MAE %.4f" % (e_tex, e_vert))
    assert e_tex <= QUALITY_BOUND < e_vert


def test_golden_fixture():
    g = np.load(os.path.join(HERE, "golden", "tiny_texture.npz"))
    s, col, m, rt, cam = _tiny_inputs()
    assert m["faces"].tobytes() == g["faces"].tobytes()
    for k, (S, K) in enumerate(g["cases"]):
        b = tr.bake(m, s["depth"], col, rt, cam, int(S), float(g["occlusion"]), int(K))
        assert b["image"].tobytes() == g[f"{k}_image"].tobytes() and b["uv"].tobytes() == g[f"{k}_uv"].tobytes(), k
        assert [b["info"][c] for c in tr.INFO_COUNTS] == g[f"{k}_info"].tolist(), k
