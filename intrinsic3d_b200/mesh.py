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


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
              "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _ply_header(data: bytes):
    """(format, elements, body offset) of a PLY file; elements: [(name, count, [(name, type) or (name, (count type, item type))])]"""
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError("load_ply: not a PLY file (no 'ply' magic or no end_header)")
    nl = data.find(b"\n", end)
    body = len(data) if nl < 0 else nl + 1
    fmt, elements = None, []
    for line in data[:end].decode("ascii", "replace").splitlines()[1:]:
        t = line.split()
        if not t or t[0] in ("comment", "obj_info"):
            continue
        if t[0] == "format":
            fmt = t[1]
        elif t[0] == "element":
            elements.append((t[1], int(t[2]), []))
        elif t[0] == "property" and elements:
            if t[1] == "list":
                if t[2] not in _PLY_TYPES or t[3] not in _PLY_TYPES:
                    raise ValueError(f"load_ply: unknown list types in {line!r}")
                elements[-1][2].append((t[4], (_PLY_TYPES[t[2]], _PLY_TYPES[t[3]])))
            elif t[1] in _PLY_TYPES:
                elements[-1][2].append((t[2], _PLY_TYPES[t[1]]))
            else:
                raise ValueError(f"load_ply: unknown property type in {line!r}")
    if fmt not in ("ascii", "binary_little_endian"):
        raise ValueError(f"load_ply: format {fmt!r} is not supported (ascii or binary_little_endian)")
    return fmt, elements, body


def load_ply(path):
    """Reads a triangle mesh from a PLY file: what save_ply writes, and ASCII or binary little-endian PLY with float or double x, y, z
    and a vertex_indices (or vertex_index) list per face; other properties and elements are skipped, and red, green, blue become the
    colours when present.  Raises ValueError for a face that is not a triangle, a missing vertex position or face list, and an index
    outside the vertices.  Returns the dict extract_mesh returns: vertices float32 [V, 3], colors uint8 [V, 3], faces int32 [F, 3], so
    load_ply -> Engine.upload_reference_mesh -> Engine.grid_from_mesh brings a mesh file in."""
    with open(path, "rb") as fh:
        data = fh.read()
    fmt, elements, pos = _ply_header(data)
    out = {}
    tokens = data[pos:].split() if fmt == "ascii" else None
    ti = 0
    for name, count, props in elements:
        is_list = [isinstance(t, tuple) for _, t in props]
        if fmt == "ascii":
            if not any(is_list):
                n = len(props) * count
                vals = np.array(tokens[ti:ti + n], np.float64).reshape(count, len(props))
                ti += n
                rec = {p: vals[:, k] for k, (p, _) in enumerate(props)}
            else:
                rec = {p: [] for p, _ in props}
                for _ in range(count):
                    for p, t in props:
                        if isinstance(t, tuple):
                            k = int(tokens[ti])
                            rec[p].append([int(x) for x in tokens[ti + 1:ti + 1 + k]])
                            ti += 1 + k
                        else:
                            rec[p].append(float(tokens[ti]))
                            ti += 1
        else:
            if sum(is_list) > 1 or (any(is_list) and name != "face"):
                raise ValueError(f"load_ply: element {name!r} with list properties is not supported in binary files")
            # every list is read as a triangle (count 3); the counts are checked below, and the first count that is not 3 is read where
            # it lies, because the records before it have the triangle size
            dt = []
            for p, t in props:
                dt += [(p + "#n", "<" + t[0]), (p, "<" + t[1], 3)] if isinstance(t, tuple) else [(p, "<" + t)]
            dt = np.dtype(dt)
            if len(data) - pos < dt.itemsize * count:
                raise ValueError(f"load_ply: element {name!r} is truncated or has faces that are not triangles")
            arr = np.frombuffer(data, dt, count, pos)
            pos += dt.itemsize * count
            rec = {p: arr[p] for p, _ in props}
            for p, t in props:
                if isinstance(t, tuple) and count and (arr[p + "#n"] != 3).any():
                    raise ValueError(f"load_ply: {name} {int(np.argmax(arr[p + '#n'] != 3))} is not a triangle")
        out[name] = (count, rec)
    if "vertex" not in out or not all(k in out["vertex"][1] for k in "xyz"):
        raise ValueError("load_ply: no vertex element with x, y, z")
    V, vr = out["vertex"]
    verts = np.stack([np.asarray(vr[k], np.float64) for k in "xyz"], 1).astype(np.float32).reshape(V, 3)
    cols = (np.stack([np.asarray(vr[k]) for k in ("red", "green", "blue")], 1).astype(np.uint8) if all(k in vr for k in ("red", "green", "blue"))
            else np.zeros((V, 3), np.uint8))
    F, fr = out.get("face", (0, {}))
    key = "vertex_indices" if "vertex_indices" in fr else ("vertex_index" if "vertex_index" in fr else None)
    if key is None:
        raise ValueError("load_ply: no face element with a vertex_indices or vertex_index list")
    lists = fr[key]
    if fmt == "ascii":
        bad = [i for i, lst in enumerate(lists) if len(lst) != 3]
        if bad:
            raise ValueError(f"load_ply: face {bad[0]} is not a triangle ({len(lists[bad[0]])} vertices)")
    faces = np.asarray(lists, np.int64).reshape(F, 3)
    if F and (faces.min() < 0 or faces.max() >= V):
        raise ValueError("load_ply: a face index lies outside the vertices")
    return dict(vertices=verts, colors=cols, faces=faces.astype(np.int32))


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
