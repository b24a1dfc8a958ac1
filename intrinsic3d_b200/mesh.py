"""Mesh output: Mesh::save of the reference (libintrinsic3d/src/mesh.cpp:41-100), byte for byte.

A mesh is the dict Engine.extract_mesh returns: vertices float32 [V, 3], colors uint8 [V, 3], faces int32 [F, 3].
"""
from __future__ import annotations

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
