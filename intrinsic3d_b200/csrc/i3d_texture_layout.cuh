/*
 * i3d_texture_layout.cuh — the per-face UV corners, the clamped barycentric map and the texel-to-point rule of the texture atlas
 * (DESIGN.md §6t; the layout and its no-bleed property are stated in i3d_texture.cuh), shared by the bake and the decomposition
 * (i3d_texture.cuh) and the rasterizer's texture lookup (i3d_raster.cuh).  No kernels.
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

// The point P and unit face normal n of local texel (i, j) of face A or B (faceB) with vertex indices fv into vpos: (a, b) = tex_bary at
// the texel centre, w0 = (1 - a) - b, P = (w0 p0 + a p1) + b p2 per coordinate; n = (v1 - v0) x (v2 - v0), each component (e1[p] e2[q]) -
// (e1[q] e2[p]), over __fsqrt_rn((n0 n0 + n1 n1) + n2 n2).  nrm is left as it is (the callers pass 0) when that length is 0.
__device__ __forceinline__ void tex_texel_point(int S, bool faceB, int i, int j, const float* vpos, int3 fv, float (&pt)[3], float (&nrm)[3])
{
    float a, b;
    tex_bary(S, faceB, static_cast<float>(i) + 0.5f, static_cast<float>(j) + 0.5f, a, b);
    const float w0 = FS(FS(1.0f, a), b);
    const float* p0 = vpos + 3 * static_cast<size_t>(fv.x);
    const float* p1 = vpos + 3 * static_cast<size_t>(fv.y);
    const float* p2 = vpos + 3 * static_cast<size_t>(fv.z);
    float e1[3], e2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        pt[k] = FA(FA(FM(w0, p0[k]), FM(a, p1[k])), FM(b, p2[k]));
        e1[k] = FS(p1[k], p0[k]); e2[k] = FS(p2[k], p0[k]);
    }
    const float n0 = FS(FM(e1[1], e2[2]), FM(e1[2], e2[1]));
    const float n1 = FS(FM(e1[2], e2[0]), FM(e1[0], e2[2]));
    const float n2 = FS(FM(e1[0], e2[1]), FM(e1[1], e2[0]));
    const float len = __fsqrt_rn(FA(FA(FM(n0, n0), FM(n1, n1)), FM(n2, n2)));
    if (len > 0.0f) { nrm[0] = FD(n0, len); nrm[1] = FD(n1, len); nrm[2] = FD(n2, len); }
}

} // namespace i3d
