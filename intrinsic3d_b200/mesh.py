"""Mesh output: Mesh::save of the reference (libintrinsic3d/src/mesh.cpp:41-100), byte for byte, and the textured OBJ of a baked texture.

A mesh is the dict Engine.extract_mesh returns: vertices float32 [V, 3], colors uint8 [V, 3], faces int32 [F, 3].  A texture is the
dict Engine.bake_texture returns: image uint8 [H, W, 3], uv float32 [F, 3, 2].
"""
from __future__ import annotations

import os
import struct
import zlib

import numpy as np


def ply_bytes(mesh) -> bytes:
    """The PLY file Mesh::save writes: an ASCII header ending each line with '\\n', then binary little-endian records, per vertex
    float x, y, z + uchar red, green, blue, per face uchar 3 + three int32 indices."""
    v = np.ascontiguousarray(mesh["vertices"], np.float32)
    c = np.ascontiguousarray(mesh["colors"], np.uint8)
    f = np.ascontiguousarray(mesh["faces"], np.int32)
    if v.ndim != 2 or v.shape[1] != 3 or c.shape != v.shape or f.ndim != 2 or f.shape[1] != 3:
        raise ValueError(f"save_ply: bad mesh shapes vertices {v.shape}, colors {c.shape}, faces {f.shape}")
    if len(v) == 0:
        raise ValueError("save_ply: the mesh has no vertices (Mesh::save refuses to write it)")
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(v)}\n"
              "property float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {len(f)}\n"
              "property list uchar int vertex_indices\n"
              "end_header\n").encode("ascii")
    vrec = np.empty(len(v), np.dtype([("p", "<f4", 3), ("c", "u1", 3)]))
    vrec["p"], vrec["c"] = v, c
    frec = np.empty(len(f), np.dtype([("n", "u1"), ("i", "<i4", 3)]))
    frec["n"], frec["i"] = 3, f
    return header + vrec.tobytes() + frec.tobytes()


def save_ply(path, mesh) -> None:
    """Writes `mesh` to `path` as Mesh::save does.  Raises ValueError for a mesh without vertices, which Mesh::save refuses."""
    data = ply_bytes(mesh)
    with open(path, "wb") as fh:
        fh.write(data)


# SDFVisualization::getOutputModes (src/sdf/visualization.cpp:72-89): settings key -> colour mode, in this order
OUTPUT_MODE_KEYS = (
    ("output_mesh_normals", "normals"),
    ("output_mesh_laplacian", "lap"),
    ("output_mesh_intensity", "lum"),
    ("output_mesh_intensity_grad", "lum_grad"),
    ("output_mesh_albedo", "albedo"),
    ("output_mesh_shading_sv", "shading_sv"),
    ("output_mesh_shading_sv_const", "shading_sv_const"),
    ("output_mesh_chromacity", "chroma"),
    ("output_mesh_subvolumes", "subvol"),
    ("output_mesh_subvolumes_interpolated", "subvol_interp"),
)


def _setting_true(v) -> bool:
    """Settings::get<bool>: the yml stores "0" / "1", read with operator>>; only 1 is true."""
    if isinstance(v, bool):
        return v
    try:
        return int(str(v).strip()) == 1
    except ValueError:
        return False


def output_modes(settings, add_voxel_colors: bool = True):
    """The colour modes of the meshes to write, as SDFVisualization::getOutputModes lists them: "" (the voxel colours) first when
    add_voxel_colors, then each mode whose key is present in `settings` (a mapping such as the loaded data/intrinsic3d.yml) and true.
    May include the subvolume modes "subvol" / "subvol_interp", which export_meshes refuses."""
    modes = [""] if add_voxel_colors else []
    modes += [mode for key, mode in OUTPUT_MODE_KEYS if key in settings and _setting_true(settings[key])]
    return modes


def mesh_file(prefix: str, mode: str) -> str:
    """SDFVisualization::exportMesh's file name: prefix, "_" + mode unless the mode is "", ".ply"."""
    return prefix + ("_" + mode if mode else "") + ".ply"


def export_meshes(engine, prefix: str, modes, largest_component_only: bool = False, source: str = "refined", cell_size=None):
    """SDFVisualization::colorize + exportMesh for every mode in `modes`: extracts the mesh of the engine's grid coloured in that mode on
    the device and writes it to mesh_file(prefix, mode).  Returns the paths written.  Every mode is checked before anything is extracted:
    the subvolume modes are refused (the reference colours subvolumes with random colours, so there is nothing reproducible to write).
    With a cell_size (metres), each mesh is simplified on the device (Engine.simplify_mesh) before it is written."""
    from .engine import COLOR_MODES
    bad = [m for m in modes if m not in COLOR_MODES]
    if bad:
        raise ValueError(f"export_meshes: unsupported colour modes {bad} (supported: {sorted(COLOR_MODES)})")
    paths = []
    for mode in modes:
        path = mesh_file(prefix, mode)
        m = engine.extract_mesh(source, largest_component_only, mode)
        if cell_size is not None:
            m = engine.simplify_mesh(cell_size)
        save_ply(path, m)
        paths.append(path)
    return paths


def png_bytes(image) -> bytes:
    """An 8-bit RGB PNG of image uint8 [H, W, 3]: every scanline with filter 0, one IDAT of zlib level 6, so equal images give equal
    bytes."""
    img = np.ascontiguousarray(image, np.uint8)
    if img.ndim != 3 or img.shape[2] != 3 or img.shape[0] == 0 or img.shape[1] == 0:
        raise ValueError(f"png_bytes: need a non-empty uint8 [H, W, 3] image, got {img.shape}")
    H, W = img.shape[:2]

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    raw = np.concatenate([np.zeros((H, 1), np.uint8), img.reshape(H, 3 * W)], axis=1).tobytes()
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw, 6))
            + chunk(b"IEND", b""))


def obj_bytes(mesh, uv, mtl_name: str) -> bytes:
    """A Wavefront OBJ of `mesh` with per-corner texture coordinates uv [F, 3, 2]: "mtllib <mtl_name>", "usemtl texture", one "v x y z"
    per vertex (%.9g, which round-trips a float32), one "vt u v" per face corner (corner k of face f is vt 3 f + k + 1) and
    "f a/t b/t c/t" with 1-based indices."""
    v = np.ascontiguousarray(mesh["vertices"], np.float32)
    f = np.ascontiguousarray(mesh["faces"], np.int64)
    t = np.ascontiguousarray(uv, np.float32)
    if v.ndim != 2 or v.shape[1] != 3 or f.ndim != 2 or f.shape[1] != 3 or t.shape != (len(f), 3, 2):
        raise ValueError(f"obj_bytes: bad shapes vertices {v.shape}, faces {f.shape}, uv {t.shape}")
    lines = [f"mtllib {mtl_name}", "usemtl texture"]
    lines += ["v %.9g %.9g %.9g" % (float(a), float(b), float(c)) for a, b, c in v]
    lines += ["vt %.9g %.9g" % (float(a), float(b)) for a, b in t.reshape(-1, 2)]
    k = 3 * np.arange(len(f), dtype=np.int64)[:, None] + np.arange(1, 4)[None, :]
    lines += ["f %d/%d %d/%d %d/%d" % (a + 1, ta, b + 1, tb, c + 1, tc) for (a, b, c), (ta, tb, tc) in zip(f.tolist(), k.tolist())]
    return ("\n".join(lines) + "\n").encode("ascii")


def save_textured_obj(prefix: str, mesh, texture):
    """Writes prefix.obj (obj_bytes), prefix.mtl (material "texture", diffuse map prefix.png) and prefix.png (png_bytes of the atlas).
    Returns the three paths."""
    base = os.path.basename(prefix)
    paths = (prefix + ".obj", prefix + ".mtl", prefix + ".png")
    mtl = f"newmtl texture\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nd 1\nillum 1\nmap_Kd {base}.png\n".encode("ascii")
    for path, data in zip(paths, (obj_bytes(mesh, texture["uv"], base + ".mtl"), mtl, png_bytes(texture["image"]))):
        with open(path, "wb") as fh:
            fh.write(data)
    return paths
