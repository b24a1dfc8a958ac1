"""Synthetic hashed-SDF scenes for parity tests and the benchmark (SURVEY.md §8d).

A bumpy sphere (radius rho0*(1+bump*sin(6*theta)*sin(5*phi))) lit by a 9-term
un-normalised SH environment (basis order of the reference,
libintrinsic3d/include/nv/shading.h:57-65), with a 3-D checker albedo, observed
by F pinhole cameras on a helix looking at the centre.  The function emits the
flat arrays that both the H100 engine (i3d_upload_*) and the CPU oracle consume:

    xyz[n,3] int32, sdf0/sdf_refined/albedo[n] f64, weight[n] f32, rgb[n,3] u8,
    lum/depth[F,H,W] f32 (already at the pyramid level used), poses[F,6] f64
    (world->camera angle-axis + translation, Q12), intr[4], dist[5], sh[n,9] f64.

Voxels are emitted in 8^3-brick-major order (brick z,y,x then local z,y,x) so that
stencil neighbours are close in memory; this order is the canonical "iteration
order" of the problem (what the reference gets from its unordered_map).

All heavy lifting is done with torch on `device` (cuda on the GPU box, cpu in tests).
"""
from __future__ import annotations

import math

import numpy as np
import torch


def _rho(d: torch.Tensor, rho0: float, bump: float) -> torch.Tensor:
    theta = torch.acos(torch.clamp(d[..., 2], -1.0, 1.0))
    phi = torch.atan2(d[..., 1], d[..., 0])
    return rho0 * (1.0 + bump * torch.sin(6.0 * theta) * torch.sin(5.0 * phi))


def _implicit(p: torch.Tensor, centre: torch.Tensor, rho0: float, bump: float) -> torch.Tensor:
    q = p - centre
    r = torch.linalg.norm(q, dim=-1)
    d = q / torch.clamp(r, min=1e-12)[..., None]
    return r - _rho(d, rho0, bump)


def _normal(p, centre, rho0, bump, h=1e-5):
    g = []
    for k in range(3):
        e = torch.zeros(3, dtype=p.dtype, device=p.device)
        e[k] = h
        g.append((_implicit(p + e, centre, rho0, bump) - _implicit(p - e, centre, rho0, bump)) / (2 * h))
    g = torch.stack(g, dim=-1)
    return g / torch.linalg.norm(g, dim=-1, keepdim=True)


def sh_basis(n: torch.Tensor) -> torch.Tensor:
    x, y, z = n[..., 0], n[..., 1], n[..., 2]
    return torch.stack([torch.ones_like(x), y, z, x, x * y, y * z, -x * x - y * y + 2 * z * z, x * z, x * x - y * y], dim=-1)


def _albedo_truth(p: torch.Tensor, cell: float) -> torch.Tensor:
    c = torch.floor(p / cell).to(torch.int64).sum(dim=-1) & 1
    return torch.where(c == 0, 0.4, 0.8).to(p.dtype)


def _rotation_to_aa(R: np.ndarray) -> np.ndarray:
    c = (np.trace(R) - 1.0) * 0.5
    c = min(1.0, max(-1.0, c))
    angle = math.acos(c)
    if angle < 1e-12:
        return np.zeros(3)
    ax = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / (2.0 * math.sin(angle))
    return ax * angle


def aa_to_rotation(w: np.ndarray) -> np.ndarray:
    th = np.linalg.norm(w)
    if th < 1e-300:
        return np.eye(3)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * (K @ K)


def make_scene(radius_vox: float = 24.0,
               voxel_size: float = 0.004,
               frames: int = 8,
               width: int = 640,
               height: int = 480,
               band: float = 3.0,
               dense_dim: int | None = None,
               bump: float = 0.03,
               sdf_noise: float = 0.1,
               pose_noise: tuple = (0.002, 0.001),
               sh_mode: str = "global",
               thin_shell_factor: float = 2.0,
               seed: int = 1,
               device: str = "cpu",
               brick_order: bool = True,
               albedo_const: float | None = None):
    """Build a synthetic scene.

    radius_vox : sphere radius in voxels (N ~ 4*pi*R^2 * 2*band for the hashed case)
    band       : hash holds every voxel with |sdf| <= band*voxel_size (the state of the
                 reference grid after clearVoxelsOutsideThinShell is a shell of about this size)
    dense_dim  : if given, the hash holds ALL dense_dim^3 voxels (config C1, "dense")
    sh_mode    : "global" (one 9-vector) or "varying" (smooth per-voxel variation, like
                 interpolated subvolume SH)
    albedo_const : if given, the true albedo is this constant instead of the 3-D checker (synthetic-truth tests: no albedo edges)
    """
    dev = torch.device(device)
    f64 = torch.float64
    vs = float(np.float32(voxel_size))              # float voxel size widened (Q15)
    rho0 = radius_vox * vs
    gen = torch.Generator(device="cpu").manual_seed(seed)

    # ------------------------------------------------------------------ voxels
    if dense_dim is not None:
        half = dense_dim // 2
        lo, hi = 0, dense_dim
        centre_v = np.array([half, half, half], dtype=np.float64)
    else:
        ext = int(math.ceil(radius_vox * (1 + bump) + band + 2))
        lo, hi = -ext, ext + 1
        centre_v = np.zeros(3)
    centre = torch.tensor(centre_v * vs, dtype=f64, device=dev)
    rng = torch.arange(lo, hi, device=dev, dtype=torch.int32)
    coords = []
    vals = []
    zchunk = max(1, int(4_000_000 // max(1, (hi - lo) ** 2)))
    for z0 in range(lo, hi, zchunk):
        zr = torch.arange(z0, min(hi, z0 + zchunk), device=dev, dtype=torch.int32)
        Z, Y, X = torch.meshgrid(zr, rng, rng, indexing="ij")
        c = torch.stack([X, Y, Z], dim=-1).reshape(-1, 3)
        p = c.to(f64) * vs
        f = _implicit(p, centre, rho0, bump)
        keep = torch.ones_like(f, dtype=torch.bool) if dense_dim is not None else (f.abs() <= band * vs)
        coords.append(c[keep])
        vals.append(f[keep])
    xyz = torch.cat(coords)
    sdf_true = torch.cat(vals)
    n = xyz.shape[0]

    if brick_order:
        b = torch.div(xyz - lo, 8, rounding_mode="floor").to(torch.int64)
        l = (xyz - lo).to(torch.int64) - b * 8
        nb = (hi - lo + 7) // 8 + 1
        key = (((b[:, 2] * nb + b[:, 1]) * nb + b[:, 0]) * 512) + (l[:, 2] * 64 + l[:, 1] * 8 + l[:, 0])
        order = torch.argsort(key)
        xyz = xyz[order]
        sdf_true = sdf_true[order]

    noise = (torch.rand(n, generator=gen, dtype=f64) - 0.5).to(dev) * 2.0 * sdf_noise * vs
    sdf = sdf_true + noise
    pv = xyz.to(f64) * vs
    # closest surface point (radial projection) for voxel colours / SH variation
    q = pv - centre
    d = q / torch.clamp(torch.linalg.norm(q, dim=-1, keepdim=True), min=1e-12)
    ps = centre + d * _rho(d, rho0, bump)[..., None]

    # ------------------------------------------------------------------ lighting
    sh0 = torch.zeros(9, dtype=f64)
    sh0[0] = 0.8
    sh0[1:] = (torch.rand(8, generator=gen, dtype=f64) - 0.5) * 0.3
    sh0 = sh0.to(dev)
    if sh_mode == "varying":
        # smooth spatial variation (3 "bands" across the object), like interpolated subvolume SH
        ph = ps / max(rho0, 1e-9)
        mod = torch.stack([torch.sin(1.5 * ph[:, 0] + k) * torch.cos(1.1 * ph[:, 1] - 0.5 * k) * torch.sin(0.7 * ph[:, 2] + 0.3 * k)
                           for k in range(9)], dim=-1)
        sh = sh0[None, :] + 0.05 * mod
    else:
        sh = sh0[None, :].expand(n, 9).clone()

    def sh_at(p_world):
        if sh_mode == "varying":
            ph = (p_world) / max(rho0, 1e-9)
            mod = torch.stack([torch.sin(1.5 * ph[..., 0] + k) * torch.cos(1.1 * ph[..., 1] - 0.5 * k) * torch.sin(0.7 * ph[..., 2] + 0.3 * k)
                               for k in range(9)], dim=-1)
            return sh0 + 0.05 * mod
        return sh0.expand(*p_world.shape[:-1], 9)

    cell = max(6.0 * vs, rho0 / 4.0)
    n_s = _normal(ps, centre, rho0, bump)
    a_s = _albedo_truth(ps - centre, cell) if albedo_const is None else torch.full((n,), float(albedo_const), dtype=f64, device=dev)
    shade_s = (sh_basis(n_s) * sh_at(ps)).sum(-1)
    grey = torch.clamp(a_s * shade_s, 0.0, 1.0)
    tint = torch.tensor([1.0, 0.92, 0.85], dtype=f64, device=dev)
    rgb = torch.clamp(torch.round(grey[:, None] * tint[None, :] * 255.0), 1, 255).to(torch.uint8)

    # ------------------------------------------------------------------ cameras
    fx = 525.0 * width / 640.0
    fy = 525.0 * height / 480.0
    cx = (width - 1) * 0.5
    cy = (height - 1) * 0.5
    dist_cam = fx * rho0 * (1 + bump) / (0.36 * height)
    poses_true = np.zeros((frames, 6))
    cen = centre.cpu().numpy()
    for f in range(frames):
        az = 2.0 * math.pi * f / frames
        el = 0.35 * math.sin(2.0 * math.pi * (f * 3 % max(frames, 1)) / max(frames, 1) + 0.3)
        Cw = cen + dist_cam * np.array([math.cos(el) * math.sin(az), math.sin(el), -math.cos(el) * math.cos(az)])
        zc = (cen - Cw)
        zc /= np.linalg.norm(zc)
        up = np.array([0.0, -1.0, 0.0])
        xc = np.cross(-up, zc)
        xc /= np.linalg.norm(xc)
        yc = np.cross(zc, xc)
        R = np.stack([xc, yc, zc], axis=0)          # world -> camera
        t = -R @ Cw
        poses_true[f, :3] = _rotation_to_aa(R)
        poses_true[f, 3:] = t

    # ------------------------------------------------------------------ render
    lum = torch.zeros((frames, height, width), dtype=torch.float32, device=dev)
    depth = torch.zeros((frames, height, width), dtype=torch.float32, device=dev)
    us = (torch.arange(width, device=dev, dtype=f64) - cx) / fx
    vsn = (torch.arange(height, device=dev, dtype=f64) - cy) / fy
    V, Ugrid = torch.meshgrid(vsn, us, indexing="ij")
    dirs_c = torch.stack([Ugrid, V, torch.ones_like(Ugrid)], dim=-1).reshape(-1, 3)
    Rb = rho0 * (1 + bump) * 1.001
    for f in range(frames):
        R = torch.tensor(aa_to_rotation(poses_true[f, :3]), dtype=f64, device=dev)
        t = torch.tensor(poses_true[f, 3:], dtype=f64, device=dev)
        o = -(R.T @ t)
        dw = dirs_c @ R                      # R^T d  (row-vector form)
        dn = torch.linalg.norm(dw, dim=-1)
        du = dw / dn[:, None]
        oc = o - centre
        bq = (du * oc).sum(-1)
        cq = (oc * oc).sum() - Rb * Rb
        disc = bq * bq - cq
        hit = disc > 0
        idx = torch.nonzero(hit).squeeze(-1)
        if idx.numel() == 0:
            continue
        duh = du[idx]
        sq = torch.sqrt(disc[idx])
        tt = -bq[idx] - sq
        t_exit = -bq[idx] + sq
        alive = torch.ones_like(tt, dtype=torch.bool)
        for _ in range(48):
            p = o + duh * tt[:, None]
            fv = _implicit(p, centre, rho0, bump)
            tt = torch.where(alive, tt + 0.7 * fv, tt)
            alive = alive & (tt < t_exit)
        p = o + duh * tt[:, None]
        fv = _implicit(p, centre, rho0, bump)
        ok = alive & (fv.abs() < 1e-7 * max(1.0, rho0 / 0.1))
        idx = idx[ok]
        p = p[ok]
        nn = _normal(p, centre, rho0, bump)
        a = _albedo_truth(p - centre, cell) if albedo_const is None else torch.full((p.shape[0],), float(albedo_const), dtype=f64, device=dev)
        val = a * (sh_basis(nn) * sh_at(p)).sum(-1)
        zcam = (p @ R.T + t)[:, 2]
        lum[f].view(-1)[idx] = val.to(torch.float32)
        depth[f].view(-1)[idx] = zcam.to(torch.float32)

    # initial (noisy) poses the optimiser starts from
    pn = torch.randn((frames, 6), generator=gen, dtype=f64).numpy()
    poses = poses_true.copy()
    poses[:, :3] += pn[:, :3] * pose_noise[0]
    poses[:, 3:] += pn[:, 3:] * pose_noise[1]

    out = dict(
        xyz=xyz.cpu().numpy().astype(np.int32),
        sdf0=sdf.cpu().numpy().copy(),
        sdf_refined=sdf.cpu().numpy().copy(),        # SDFAlgorithms::convert: sdf_refined = sdf
        sdf_true=sdf_true.cpu().numpy(),
        albedo=np.full(n, 0.6, np.float64),          # VoxelSBR default
        albedo_true=a_s.cpu().numpy(),               # ground-truth albedo at the closest surface point (KA3 tests)
        weight=np.ones(n, np.float32),
        rgb=rgb.cpu().numpy(),
        voxel_size=np.float32(voxel_size),
        lum=lum.cpu().numpy(),
        depth=depth.cpu().numpy(),
        pyr_scale=1.0,
        poses=poses,
        poses_true=poses_true,
        intr=np.array([fx, fy, cx, cy], np.float64),
        dist=np.zeros(5, np.float64),
        sh=sh.cpu().numpy().copy(),
        thres_shell=float(thin_shell_factor) * float(np.float32(voxel_size)),
    )
    return out


# BASELINE.json configs -> generator arguments (N is the number of hash entries)
def make_color_frames(scene, seed: int = 7):
    """Synthetic colour frames for the recolouring pass: uint8 [F, H, W, 3] in the reference's cv::Mat channel order (B, G, R),
    derived from the rendered luminance with a tint and a smooth per-frame chroma pattern so the three channels differ."""
    lum = np.asarray(scene["lum"], np.float32)
    F, H, W = lum.shape
    rng = np.random.default_rng(seed)
    xx = np.arange(W, dtype=np.float32)[None, :]
    yy = np.arange(H, dtype=np.float32)[:, None]
    out = np.empty((F, H, W, 3), np.uint8)
    for f in range(F):
        ph = rng.uniform(0, 2 * np.pi, 3).astype(np.float32)
        base = lum[f] * np.float32(255.0)
        lit = lum[f] > 0
        chans = (base * (np.float32(0.85) + np.float32(0.07) * np.sin((xx + yy) / np.float32(53.0) + ph[2])),      # B
                 base * (np.float32(0.92) + np.float32(0.05) * np.cos(yy / np.float32(29.0) + ph[1])),             # G
                 base * (np.float32(1.00) + np.float32(0.06) * np.sin(xx / np.float32(37.0) + ph[0])))             # R
        for k, ch in enumerate(chans):
            out[f, :, :, k] = np.clip(np.rint(np.where(lit, ch, np.float32(12.0))), 0, 255).astype(np.uint8)
    return out


def _latlong(n_theta: int):
    """unit-sphere directions on n_theta rings of latitude (the two poles included) by 2 n_theta meridians, and the faces between them:
    a fan at each pole, two triangles per quad elsewhere (2 n_theta (2 n_theta - 2) faces)"""
    n_phi = 2 * n_theta
    th = np.arange(1, n_theta) * (math.pi / n_theta)
    ph = np.arange(n_phi) * (2.0 * math.pi / n_phi)
    T, P = np.meshgrid(th, ph, indexing="ij")
    ring = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)
    d = np.concatenate([[[0.0, 0.0, 1.0]], ring, [[0.0, 0.0, -1.0]]])
    south = len(d) - 1
    j = np.arange(n_phi)
    jn = (j + 1) % n_phi
    idx = lambda i, jj: 1 + i * n_phi + jj          # noqa: E731  ring i (0 .. n_theta - 2), meridian jj
    faces = [np.stack([np.zeros_like(j), idx(0, j), idx(0, jn)], 1)]
    for i in range(n_theta - 2):
        faces.append(np.stack([idx(i, j), idx(i + 1, j), idx(i + 1, jn)], 1))
        faces.append(np.stack([idx(i, j), idx(i + 1, jn), idx(i, jn)], 1))
    faces.append(np.stack([np.full_like(j, south), idx(n_theta - 2, jn), idx(n_theta - 2, j)], 1))
    return d, np.concatenate(faces)


def _truth_geometry(radius_vox=24.0, voxel_size=0.004, band=3.0, dense_dim=None, bump=0.03, **_):
    """rho0, centre and bump exactly as make_scene computes them (the other make_scene arguments do not move the surface)"""
    vs = float(np.float32(voxel_size))
    rho0 = radius_vox * vs
    centre_v = np.array([dense_dim // 2] * 3, np.float64) if dense_dim is not None else np.zeros(3)
    return rho0, centre_v * vs, bump, vs


def truth_mesh(n_theta: int | None = None, **geometry):
    """The analytic surface of make_scene as a fine triangle mesh: every vertex of a latitude-longitude grid of directions d at
    centre + d rho(d).  The bump's sin(6 theta) sin(5 phi) has a cone-like point at each pole; the grid puts a vertex there and a fan of
    2 n_theta thin faces around it, which follows it closely.  geometry: make_scene's (or config_geometry's) arguments; only
    radius_vox, voxel_size, dense_dim and bump matter.  n_theta: the rings (2 n_theta (2 n_theta - 2) faces); None picks the smallest
    power of two >= 128 whose ring spacing is at most a voxel.  Returns a dict with vertices float32 [V, 3], faces int32 [F, 3] and colors
    uint8 [V, 3] (zero), the shape of an extract_mesh dict.  truth_mesh_error states how far it lies from the analytic surface."""
    rho0, centre, bump, vs = _truth_geometry(**geometry)
    if n_theta is None:
        n_theta = 128
        while math.pi * rho0 * (1 + bump) / n_theta > vs:
            n_theta *= 2
    d, f = _latlong(n_theta)
    v = centre[None, :] + d * _rho(torch.from_numpy(d), rho0, bump).numpy()[:, None]
    return dict(vertices=v.astype(np.float32), faces=f.astype(np.int32), colors=np.zeros((len(v), 3), np.uint8))


def truth_mesh_error(mesh, **geometry):
    """The largest |implicit| of make_scene's surface (metres, float64) at the face centroids and edge midpoints of the float32 mesh:
    a bound on how far the tessellation lies from the analytic surface where it is furthest from its vertices"""
    rho0, centre, bump, _ = _truth_geometry(**geometry)
    v = np.asarray(mesh["vertices"], np.float64)
    f = np.asarray(mesh["faces"], np.int64)
    pts = [(v[f[:, 0]] + v[f[:, 1]] + v[f[:, 2]]) / 3.0] + [(v[f[:, k]] + v[f[:, (k + 1) % 3]]) / 2.0 for k in range(3)]
    c = torch.tensor(centre, dtype=torch.float64)
    return max(float(_implicit(torch.from_numpy(p), c, rho0, bump).abs().max()) for p in pts)


def config_geometry(name: str):
    """make_scene's arguments of config_scene(name): what truth_mesh(**config_geometry(name)) takes"""
    return dict(_PRESETS[name])


def config_scene(name: str, device: str = "cpu", **over):
    kw = dict(_PRESETS[name])
    kw.update(over)
    return make_scene(device=device, **kw)


# config name -> make_scene arguments (N is the number of hash entries)
_PRESETS = {
    # C1: 64^3 dense, 8 frames
    "c1": dict(dense_dim=64, radius_vox=24.0, frames=8, voxel_size=0.004),
    # small hashed case for fast CPU tests
    "tiny": dict(radius_vox=10.0, frames=6, width=160, height=120, voxel_size=0.004),
    "small": dict(radius_vox=20.0, frames=8, width=320, height=240, voxel_size=0.004),
    # C2: ~500 K voxels, 50 frames      (N = 4*pi*R^2*2*band => R ~ 81.5 at band 3)
    "c2": dict(radius_vox=81.4, frames=50, voxel_size=0.002),
    # C3: ~2 M voxels, 200 frames, spatially varying SH
    "c3": dict(radius_vox=162.9, frames=200, voxel_size=0.002, sh_mode="varying"),
}
