"""CPU tests of the texture decomposition and the relit raster's restatement (tests/intrinsic_texture_ref.py, DESIGN.md §6x): known
answers of the decomposition, the relit colour against the albedo image and against the texture source, and lookups that read only
owned texels."""
import numpy as np

import intrinsic_texture_ref as it
import raster_ref as ra
import texture_ref as tr
from intrinsic3d_b200.mesh import albedo_image

f32 = np.float32
EYE = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], f32)
CAM = dict(fx=f32(40.0), fy=f32(40.0), cx=f32(15.5), cy=f32(11.5), d=np.zeros(5, f32))
W, H = 32, 24
SH = np.array([0.8, 0.1, -0.15, 0.2, 0.05, -0.03, 0.04, 0.02, -0.06], f32)


def _mesh(V, F):
    V = np.asarray(V, f32).reshape(-1, 3)
    return dict(vertices=V, faces=np.asarray(F, np.int32).reshape(-1, 3), colors=np.full((len(V), 3), 90, np.uint8))


def _quad(z=2.0, s=0.45):
    """two faces facing the camera of EYE / CAM: faces 0 and 1 share cell 0"""
    return _mesh([[-s * z, -s * z, z], [s * z, -s * z, z], [s * z, s * z, z], [-s * z, s * z, z]], [[0, 1, 2], [0, 2, 3]])


def _image(mesh, S, colour):
    L = tr.layout(len(mesh["faces"]), S)
    tp = tr.texel_points(mesh, S)
    img = np.zeros((L["H"], L["W"], 3), np.uint8)
    img[tp["y"], tp["x"]] = np.asarray(colour, np.uint8)
    return img, tp


def test_constant_colour_on_a_flat_face_known_answer():
    S, c = 10, (200, 120, 40)
    m = _quad()
    img, tp = _image(m, S, c)
    r = it.decompose(img, m, S, it.global_sh(SH))
    n = tp["N"][0]
    assert np.all(tp["N"] == n) and abs(float(np.linalg.norm(n)) - 1) < 1e-6
    s = it.sh_dot(n[None], SH[None])[0]
    assert s > 0.05
    want = [(f32(ck) / f32(255)) / s for ck in c]                    # one rounded division each, in that order
    a = r["albedo"][tp["y"], tp["x"]]
    assert all(np.all(a[:, k] == f32(want[k])) for k in range(3))
    assert np.all(r["shading"][tp["y"], tp["x"]] == s)
    own = np.zeros(img.shape[:2], bool)
    own[tp["y"], tp["x"]] = True
    assert np.all(r["albedo"][~own] == 0) and np.all(r["shading"][~own] == 0)
    i = r["info"]
    assert i["num_texels_owned"] == 2 * S * (S - 1) // 2 == i["num_texels_lit"] and i["num_texels_unlit"] == 0
    assert i["albedo_min"] == i["albedo_max"] == [float(f32(w)) for w in want]


def test_low_shading_and_zero_area_faces_give_zero():
    S = 8
    m = _quad()
    img, tp = _image(m, S, (100, 100, 100))
    s = it.sh_dot(tp["N"][:1], SH[None])[0]
    r = it.decompose(img, m, S, it.global_sh(SH), min_shading=float(s))      # s <= min_shading: unlit
    assert r["info"]["num_texels_lit"] == 0 and not r["albedo"].any() and r["shading"][tp["y"], tp["x"]].min() == s
    dark = it.decompose(img, m, S, it.global_sh(-SH))                      # negative shading
    assert dark["info"]["num_texels_unlit"] == dark["info"]["num_texels_owned"] and not dark["albedo"].any()
    flat = _mesh([[0, 0, 2], [0.5, 0, 2], [1.0, 0, 2], [0, 0.5, 2]], [[0, 1, 2], [0, 1, 3]])       # face 0 has zero area
    img, tp = _image(flat, S, (100, 100, 100))
    r = it.decompose(img, flat, S, it.global_sh(SH))
    z = tp["face"] == 0
    assert not r["albedo"][tp["y"][z], tp["x"][z]].any() and not r["shading"][tp["y"][z], tp["x"][z]].any()
    assert r["albedo"][tp["y"][~z], tp["x"][~z]].all()


def test_fallback_texels_are_decomposed_and_counted():
    S = 8
    m = _quad()
    img, tp = _image(m, S, (90, 90, 90))
    obs = np.zeros(img.shape[:2], bool)
    obs[tp["y"][tp["face"] == 0], tp["x"][tp["face"] == 0]] = True           # face 1's texels had no observation
    r = it.decompose(img, m, S, it.global_sh(SH), observed_mask=obs)
    assert r["info"]["num_texels_lit_fallback"] == int((tp["face"] == 1).sum()) > 0
    assert r["albedo"][tp["y"][tp["face"] == 1], tp["x"][tp["face"] == 1]].all()
    # with no frames at all every texel is a fallback texel
    none = it.observed(m, np.zeros((0, H, W), f32), np.zeros((0, 12), f32), CAM, S)
    assert not none.any()
    assert it.decompose(img, m, S, it.global_sh(SH), observed_mask=none)["info"]["num_texels_lit_fallback"] == r["info"]["num_texels_lit"]


def test_one_subvolume_is_taken_unblended():
    P = np.array([[0.0, 0.0, 0.0], [5.0, -3.0, 9.0]], f32)               # the second point is far from the subvolume
    sub = SH.astype(np.float64)[None] * 1.0000001
    got = it.estimate_sh(np.array([[0, 0, 0]]), sub, 0.1)(P)
    assert np.all(got == sub[0].astype(f32))
    two = it.estimate_sh(np.array([[0, 0, 0], [1, 0, 0]]), np.concatenate([sub, 2 * sub]), 0.1)(P)
    assert np.all(two[1] == 0) and np.any(two[0] != 0)


def _decomposed_quad(S=10):
    m = _quad()
    L = tr.layout(2, S)
    tp = tr.texel_points(m, S)
    rng = np.random.default_rng(5)
    img = np.zeros((L["H"], L["W"], 3), np.uint8)
    img[tp["y"], tp["x"]] = rng.integers(30, 250, (len(tp["x"]), 3))
    return m, img


def test_relit_with_the_constant_sh_is_the_albedo_image():
    S = 10
    m, img = _decomposed_quad(S)
    d = it.decompose(img, m, S, it.global_sh(SH))
    one = np.array([1, 0, 0, 0, 0, 0, 0, 0, 0], f32)
    r = it.rasterize(m, EYE[None], CAM, W, H, d["albedo"], S, it.global_sh(one))
    face = r["face"][0].reshape(-1)
    p = face >= 0
    assert p.sum() > 100
    bar = r["bary"][0].reshape(-1, 2)[p]
    _, _, X, Y = it.lookup(face[p].astype(np.int64), bar[:, 0], bar[:, 1], S, tr.layout(2, S)["cols"])
    A = np.stack([it.interp_f32(d["albedo"], X, Y, k) for k in range(3)], 1)
    assert r["rgb"][0].reshape(-1, 3)[p].tobytes() == albedo_image(A).tobytes()
    assert not r["rgb"][0].reshape(-1, 3)[~p].any()


def test_relighting_with_the_decomposition_sh_reproduces_the_texture():
    S = 10
    m, img = _decomposed_quad(S)
    d = it.decompose(img, m, S, it.global_sh(SH))
    rel = it.rasterize(m, EYE[None], CAM, W, H, d["albedo"], S, it.global_sh(SH))
    tex = ra.rasterize(m, EYE[None], CAM, W, H, color="texture", texture=(img, S))       # asserts that lookups read owned texels only
    face = tex["face"][0].reshape(-1)
    p = face >= 0
    diff = np.abs(rel["rgb"][0].reshape(-1, 3)[p].astype(int) - tex["rgb"][0].reshape(-1, 3)[p].astype(int))
    assert diff.max() <= 1 and (diff == 0).mean() > 0.5
    # and the lookups of the relit source read only texels the face owns, with every tap lit here
    bar = tex["bary"][0].reshape(-1, 2)[p]
    _, _, X, Y = it.lookup(face[p].astype(np.int64), bar[:, 0], bar[:, 1], S, 1)
    ra._texture_colour(face[p].astype(np.int64), bar[:, 0], bar[:, 1], img, S, 1)
    lit = d["shading"] > 0.05
    for dx in (0, 1):
        for dy in (0, 1):
            xx, yy = np.floor(X).astype(int) + dx, np.floor(Y).astype(int) + dy
            wx = (X - np.floor(X)) if dx else (1 - (X - np.floor(X)))
            wy = (Y - np.floor(Y)) if dy else (1 - (Y - np.floor(Y)))
            live = (wx * wy) > 0
            assert lit[np.clip(yy, 0, lit.shape[0] - 1), np.clip(xx, 0, lit.shape[1] - 1)][live].all()


def test_albedo_image_rounding():
    a = np.array([[[0.0, 0.5, 1.0], [-0.1, 1.2, 0.0019607844]]], f32)
    assert albedo_image(a).tolist() == [[[0, 128, 255], [0, 255, 1]]]
    assert albedo_image(a, 0.5)[0, 0].tolist() == [0, 64, 128]


# ---- quality on the tiny scene: does the decomposition recover reflectance? ----------------------------------------------------
G = np.array([1.00, 0.92, 0.85])            # make_color_frames' channel gains (R, G, B)


def _surface(s, P, radius_vox=10.0):
    """The scene's radially closest surface point of P: true albedo, true unit normal (float64)."""
    import torch
    from intrinsic3d_b200 import scene as sc
    vs = float(np.float32(s["voxel_size"]))
    rho0, bump = radius_vox * vs, 0.03
    p = torch.tensor(np.asarray(P, np.float64))
    d = p / torch.linalg.norm(p, dim=-1, keepdim=True)
    ps = d * sc._rho(d, rho0, bump)[..., None]
    n = sc._normal(ps, torch.zeros(3, dtype=torch.float64), rho0, bump)
    return sc._albedo_truth(ps, max(6.0 * vs, rho0 / 4.0)).numpy(), n.numpy()


def _basis(n):
    import torch
    from intrinsic3d_b200 import scene as sc
    return sc.sh_basis(torch.tensor(n)).numpy()


def _fit(est, truth):
    """est = alpha truth by least squares; returns (alpha, mean |est / alpha - truth|)."""
    alpha = float((est * truth).sum() / (truth * truth).sum())
    return alpha, float(np.abs(est / alpha - truth).mean())


_QUALITY = {}


def _quality_inputs():
    """tiny after recompute_colors, the refined mesh simplified at 4 voxels, its S = 12 texture from all keyframes and from the even ones,
    the oracle's lighting estimate"""
    if _QUALITY:
        return _QUALITY
    import mesh_ref
    import mesh_simplify_ref as msr
    import oracle
    import render_ref as rr
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    s = config_scene("tiny")
    col = make_color_frames(s)
    o = oracle.Oracle(threads=4)
    o.load_scene(s)
    o.set_color_frames(col)
    o.recompute_colors(0.02, 5)
    lp = oracle.default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    o.estimate_lighting(lp)
    idx, sub = o.lighting()
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], o.colors(), float(s["voxel_size"]), False)
    m = msr.simplify(m, 4 * float(s["voxel_size"]))
    rt, cam = rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"])
    even = np.arange(0, len(rt), 2)
    _QUALITY.update(s=s, col=col, m=m, rt=rt, cam=cam, even=even, S=12,
                    estimate=it.estimate_sh(idx, sub, float(lp.subvolume_size)), true_sh=np.asarray(s["sh"][0], np.float64),
                    all=tr.bake(m, s["depth"], col, rt, cam, 12, 0.02, 5),
                    held=tr.bake(m, s["depth"][even], col[even], rt[even], cam, 12, 0.02, 5))
    return _QUALITY


# Mean |A / alpha - a| over the owned texels lit under both lightings (A: channel mean of A_k / g_k; a: the true albedo; alpha: one
# least-squares scale), S = 12 texture of the refined mesh simplified at 4 voxels.  Measured: decomposition under the oracle's estimate
# 0.0777, under the true SH 0.0792, the colour texture itself (c / 255 / g) 0.1250.  The decomposition wins by about a third; the
# estimate does as well as the true SH because the remaining error is the texture's own (resampling, the checker's edges).
ALBEDO_BOUND = dict(estimate=0.085, true_sh=0.085, colour_at_least=0.115)


def test_decomposition_recovers_albedo_on_tiny():
    q = _quality_inputs()
    S, m, img = q["S"], q["m"], q["all"]["image"]
    tp = tr.texel_points(m, S)
    truth, _ = _surface(q["s"], tp["P"])
    de = it.decompose(img, m, S, q["estimate"])
    dt = it.decompose(img, m, S, it.global_sh(q["true_sh"].astype(f32)))
    lit = (de["albedo"][tp["y"], tp["x"]].any(1)) & (dt["albedo"][tp["y"], tp["x"]].any(1))
    assert lit.mean() > 0.9
    est = lambda a: (a[tp["y"], tp["x"]].astype(np.float64) / G).mean(1)[lit]
    colour = (img[tp["y"], tp["x"]].astype(np.float64) / 255.0 / G).mean(1)[lit]
    r = {k: _fit(v, truth[lit]) for k, v in (("estimate", est(de["albedo"])), ("true_sh", est(dt["albedo"])), ("colour", colour))}
    print("albedo MAE on tiny: " + ", ".join(f"{k} {v[1]:.4f} (scale {v[0]:.3f})" for k, v in r.items()))
    assert r["true_sh"][1] <= ALBEDO_BOUND["true_sh"] and r["estimate"][1] <= ALBEDO_BOUND["estimate"]
    assert r["colour"][1] >= ALBEDO_BOUND["colour_at_least"]
    assert max(r["estimate"][1], r["true_sh"][1]) < r["colour"][1]


# Mean |rgb - truth| per channel (uint8 units) over the covered pixels of the odd keyframes: the decomposition of the even keyframes'
# texture (oracle estimate) relit under SH' = the true SH with its band-1 terms negated, divided by the fitted albedo scale, against the
# scene's appearance under SH'; the plain texture source against the same truth.  Measured: relit 19.49, texture source 33.21 -
# relighting wins.
RELIGHT_BOUND = dict(relit=21.5, texture_at_least=30.0)


def test_relighting_on_tiny():
    q = _quality_inputs()
    S, m, img, s = q["S"], q["m"], q["held"]["image"], q["s"]
    d = it.decompose(img, m, S, q["estimate"])
    tp = tr.texel_points(m, S)
    truth, _ = _surface(s, tp["P"])
    lit = d["albedo"][tp["y"], tp["x"]].any(1)
    alpha, _ = _fit((d["albedo"][tp["y"], tp["x"]].astype(np.float64) / G).mean(1)[lit], truth[lit])
    sh2 = q["true_sh"].copy()
    sh2[1:4] = -sh2[1:4]
    odd = np.arange(1, len(q["rt"]), 2)
    _, Hh, Ww = s["depth"].shape
    rel = it.rasterize(m, q["rt"], q["cam"], Ww, Hh, d["albedo"], S, it.global_sh((sh2 / alpha).astype(f32)), ids=odd)
    tex = ra.rasterize(m, q["rt"], q["cam"], Ww, Hh, color="texture", texture=(img, S), ids=odd)
    V = m["vertices"].astype(np.float64)
    Fc = m["faces"].astype(np.int64)
    err = {"relit": [], "texture": []}
    for i in range(len(odd)):
        face = rel["face"][i].reshape(-1)
        p = np.nonzero(face >= 0)[0]
        bar = rel["bary"][i].reshape(-1, 2)[p].astype(np.float64)
        f = Fc[face[p]]
        P = (1 - bar[:, :1] - bar[:, 1:]) * V[f[:, 0]] + bar[:, :1] * V[f[:, 1]] + bar[:, 1:] * V[f[:, 2]]
        a, n = _surface(s, P)
        want = np.clip((a * (_basis(n) @ sh2))[:, None] * G[None] * 255.0, 0, 255)
        for k, o in (("relit", rel), ("texture", tex)):
            err[k].append(np.abs(o["rgb"][i].reshape(-1, 3)[p].astype(np.float64) - want))
    e = {k: float(np.concatenate(v).mean()) for k, v in err.items()}
    print("relighting on tiny (odd keyframes, uint8 MAE): relit %.2f, texture source %.2f (albedo scale %.3f)" % (e["relit"], e["texture"], alpha))
    assert e["relit"] <= RELIGHT_BOUND["relit"] and e["texture"] >= RELIGHT_BOUND["texture_at_least"] and e["relit"] < e["texture"]


def test_golden_fixture():
    """tests/golden/tiny_intrinsic_texture.npz (make_golden_intrinsic_texture.py) from the restatement."""
    import hashlib
    import os
    import mesh_ref
    import render_ref as rr
    from intrinsic3d_b200.scene import config_scene, make_color_frames
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_intrinsic_texture.npz"))
    s = config_scene("tiny")
    col = make_color_frames(s)
    m = mesh_ref.extract(s["xyz"], s["sdf_refined"], s["weight"], s["rgb"], float(s["voxel_size"]), True)
    assert m["faces"].tobytes() == g["faces"].tobytes()
    rt, cam = rr.pose_rt(s["poses"]), rr.camera(s["intr"], s["dist"])
    S, ms = 6, float(g["min_shading"])
    assert tr.bake(m, s["depth"], col, rt, cam, S, 0.02, 5)["image"].tobytes() == g["image"].tobytes()
    assert it.observed(m, s["depth"], rt, cam, S).tobytes() == g["observed"].tobytes()
    d = it.decompose(g["image"], m, S, it.global_sh(g["sh"]), ms, g["observed"])
    assert d["albedo"].tobytes() == g["global_albedo"].tobytes() and d["shading"].tobytes() == g["global_shading"].tobytes()
    assert [d["info"][k] for k in it.INFO_COUNTS] == g["global_info"].tolist()
    assert np.array([d["info"]["albedo_min"], d["info"]["albedo_max"]], f32).tobytes() == g["global_range"].tobytes()
    e = it.decompose(g["image"], m, S, it.estimate_sh(g["sub_index"], g["sub_sh"], float(g["subvolume_size"])), ms, g["observed"])
    assert hashlib.sha256(e["albedo"].tobytes() + e["shading"].tobytes()).digest() == g["estimate_digest"].tobytes()
    assert [e["info"][k] for k in it.INFO_COUNTS] == g["estimate_info"].tolist()
    _, Hh, Ww = s["depth"].shape
    r = it.rasterize(m, rt, cam, Ww, Hh, d["albedo"], S, it.global_sh(g["sh"]), depth=s["depth"], bgr=col, ids=g["relit_ids"])
    assert r["rgb"].tobytes() == g["relit_rgb"].tobytes() and r["face"].tobytes() == g["relit_face"].tobytes()
    assert [[st["num_covered"], st["color_count"], *st["color_abs"], *st["color_sq"]] for st in r["stats"]] == g["relit_counts"].tolist()
