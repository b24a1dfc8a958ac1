/*
 * i3d_vis.cuh — the per-voxel colour modes of SDFVisualization::colorize (libintrinsic3d/src/sdf/visualization.cpp:101-416) on the
 * device (DESIGN.md §6k).  One thread per voxel writes the voxel's colour in the given mode; the surface extraction then takes these
 * colours in place of the voxel colours.  Every mode reads only the voxel and its ±1 ring, never a colour another thread writes.
 *
 *   I3D_MESH_COLOR_NORMALS           applyColorNormals           (:228-240)
 *   I3D_MESH_COLOR_LAPLACIAN         applyColorLaplacian         (:243-259), SDFOperators::laplacian (src/sdf/operators.cpp:80-104)
 *   I3D_MESH_COLOR_INTENSITY         applyColorIntensity
 *   I3D_MESH_COLOR_INTENSITY_GRAD    applyColorIntensityGradient (:273-306), SDFOperators::intensityGradient (operators.cpp:107-139)
 *   I3D_MESH_COLOR_ALBEDO            applyColorAlbedo
 *   I3D_MESH_COLOR_SHADING_SV(_CONST) applyColorShading         (:318-357), Shading::computeShading (src/shading.cpp:61-73)
 *   I3D_MESH_COLOR_CHROMACITY        applyColorChromacity        (:360-371), chromacity (src/color_util.cpp:61-67)
 *
 * Compiled in the surface extraction's translation unit (i3d_mesh.cu) and launched through mesh::colorize (i3d_mesh.h).  Every float
 * operation is explicitly rounded and every uchar cast truncates, so the colours are byte-equal to tests/vis_ref.py.
 */
#pragma once
#include "i3d_grid.cuh"
#include "../../include/i3d_types.h"

namespace i3d
{

// scalarToColor (src/color_util.cpp:70-78): min(max(v * s, 0), 255), truncated.  With s == 1 the product is v itself.
__device__ __forceinline__ unsigned char vis_u8(float v) { v = v < 0.0f ? 0.0f : v; v = 255.0f < v ? 255.0f : v; return static_cast<unsigned char>(v); }
__device__ __forceinline__ unsigned char vis_u8(double v) { v = v < 0.0 ? 0.0 : v; v = 255.0 < v ? 255.0 : v; return static_cast<unsigned char>(v); }
__device__ __forceinline__ uchar4 vis_grey(unsigned char c) { return make_uchar4(c, c, c, 0); }

// SDFAlgorithms::checkVoxelsValid(collectRingNeighborhood(v)): all six ±1 neighbours exist with weight > 0
__device__ __forceinline__ bool vis_ring_valid(const GridView& g, int64_t v)
{
    bool ok = true;
#pragma unroll
    for (int o = 0; o < 6; ++o)
    {
        const int32_t nb = g.nbr[static_cast<int64_t>(o) * g.n + v];
        ok = ok && nb >= 0 && g.weight[nb] > 0.0f;
    }
    return ok;
}

// computeSurfaceNormal, and false where the reference sees n.norm() == 0 or NaN
__device__ __forceinline__ bool vis_normal(const GridView& g, int64_t v, float n[3])
{
    return surface_normal_f(g, v, n) && !(isnan(n[0]) || isnan(n[1]) || isnan(n[2]));
}

// Shading::computeShading(n, sh, albedo) on a unit normal: albedo * sh_dot(n, sh) (i3d_grid.cuh); 0 for albedo 0 or NaN.
__device__ __forceinline__ float vis_shading(const float n[3], const float sh[9], float albedo)
{
    if (albedo == 0.0f || isnan(albedo)) return 0.0f;
    return FM(albedo, sh_dot(n, sh));
}

template <int MODE>
__device__ __forceinline__ uchar4 vis_color(const GridView& g, const SubvolGrid& sg, const double* __restrict__ sub_sh, int S, int64_t v)
{
    if (MODE == I3D_MESH_COLOR_NORMALS)
    {
        float n[3];
        if (!vis_normal(g, v, n)) return make_uchar4(0, 0, 0, 0);
        unsigned char c[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) c[d] = static_cast<unsigned char>(FM(FA(FM(0.5f, n[d]), 0.5f), 255.0f));
        return make_uchar4(c[0], c[1], c[2], 0);
    }
    if (MODE == I3D_MESH_COLOR_LAPLACIAN)
    {
        if (!vis_ring_valid(g, v)) return vis_grey(0);
        const float s = static_cast<float>(g.sdf[v]), s2 = FM(2.0f, s);
        float d[3];
#pragma unroll
        for (int a = 0; a < 3; ++a)
            d[a] = FS(FA(static_cast<float>(g.sdf[g.nbr[(2 * a) * g.n + v]]), static_cast<float>(g.sdf[g.nbr[(2 * a + 1) * g.n + v]])), s2);
        const float lap = FD(FA(FA(d[0], d[1]), d[2]), g.truncation);
        return vis_grey(vis_u8(FM(FA(FM(0.5f, lap), 0.5f), 255.0f)));
    }
    if (MODE == I3D_MESH_COLOR_INTENSITY) return vis_grey(vis_u8(intensity_u8(g.rgb[v])));
    if (MODE == I3D_MESH_COLOR_INTENSITY_GRAD)
    {
        if (!vis_ring_valid(g, v)) return vis_grey(127);
        const float dx = FS(intensity_u8(g.rgb[g.nbr[NB_XP * g.n + v]]), intensity_u8(g.rgb[v]));
        return vis_grey(vis_u8(FA(FM(dx, 0.5f), 127.0f)));
    }
    if (MODE == I3D_MESH_COLOR_ALBEDO) return vis_grey(vis_u8(__dmul_rn(g.albedo[v], 255.0)));
    if (MODE == I3D_MESH_COLOR_SHADING_SV || MODE == I3D_MESH_COLOR_SHADING_SV_CONST)
    {
        float n[3];
        if (!vis_normal(g, v, n)) return make_uchar4(0, 0, 0, 0);
        float sh[9];
        if (S == 1)
        {
#pragma unroll
            for (int k = 0; k < 9; ++k) sh[k] = __double2float_rn(sub_sh[k]);
        }
        else
        {
            double avg[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) avg[k] = 0.0;
            svsh_blend(g, v, sg, sub_sh, avg);
#pragma unroll
            for (int k = 0; k < 9; ++k) sh[k] = __double2float_rn(avg[k]);
        }
        const float a = MODE == I3D_MESH_COLOR_SHADING_SV_CONST ? 0.7f : __double2float_rn(g.albedo[v]);
        const float shad = __double2float_rn(__dmul_rn(static_cast<double>(vis_shading(n, sh, a)), 255.0));
        return vis_grey(vis_u8(shad));
    }
    // I3D_MESH_COLOR_CHROMACITY
    const uchar4 rgb = g.rgb[v];
    const float lum = intensity_u8(rgb);
    const float inv = FD(1.0f, lum < 0.001f ? 0.001f : lum);
    const float c[3] = {static_cast<float>(rgb.x), static_cast<float>(rgb.y), static_cast<float>(rgb.z)};
    unsigned char o[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) o[d] = vis_u8(FM(FM(FM(c[d], inv), 255.0f), 0.5f));
    return make_uchar4(o[0], o[1], o[2], 0);
}

// One thread per voxel: the colour of voxel v in mode MODE.  g.sdf is the sdf the mesh is cut from; sg / sub_sh [S][9] are the subvolumes
// and subvolume SH of the last lighting estimate (read by the shading modes only).
template <int MODE>
__global__ void __launch_bounds__(kThreads) k_vis_colors(GridView g, SubvolGrid sg, const double* __restrict__ sub_sh, int S, uchar4* __restrict__ out)
{
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (v >= g.n) return;
    out[v] = vis_color<MODE>(g, sg, sub_sh, S, v);
}

} // namespace i3d
