/*
 * i3d_texture_layout.cuh — the per-face UV corners and the clamped barycentric map of the texture atlas (DESIGN.md §6t; the layout and
 * its no-bleed property are stated in i3d_texture.cuh), shared by the bake (i3d_texture.cuh) and the rasterizer's texture lookup
 * (i3d_raster.cuh).  No kernels.
 */
#pragma once
#include "i3d_grid.cuh"

namespace i3d
{

// UV corner k (0, 1, 2 = v0, v1, v2) of face A (b = false) or B (b = true) of a cell, in local texel units
__device__ __forceinline__ void tex_corner(int S, bool b, int k, float& u, float& v)
{
    const float base = b ? static_cast<float>(S - 1) : 1.0f;     // v0's u and v
    const float far = b ? 3.0f : static_cast<float>(S - 3);      // v1's u, v2's v
    u = k == 1 ? far : base;
    v = k == 2 ? far : base;
}

// The clamped barycentric coordinates (a, b) of local texel position (u, v) of face A or B
__device__ __forceinline__ void tex_bary(int S, bool faceB, float u, float v, float& a, float& b)
{
    const float L = static_cast<float>(S - 4);
    if (!faceB) { a = FD(FS(u, 1.0f), L); b = FD(FS(v, 1.0f), L); }
    else { const float e = static_cast<float>(S - 1); a = FD(FS(e, u), L); b = FD(FS(e, v), L); }
    a = a < 0.0f ? 0.0f : a;
    b = b < 0.0f ? 0.0f : b;
    const float s = FA(a, b);
    if (s > 1.0f) { a = FD(a, s); b = FD(b, s); }
}

} // namespace i3d
