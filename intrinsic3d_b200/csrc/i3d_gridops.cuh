/*
 * i3d_gridops.cuh — grid-level transitions on the device (SURVEY.md §8 f3): the voxel set changes between refinement levels
 * without a round trip through a host hash map.
 *
 *   k_shell_keep + k_shell_crossing  SDFAlgorithms::clearVoxelsOutsideThinShell (libintrinsic3d/src/sdf/algorithms.cpp:368-458),
 *                                    called by Intrinsic3D::prepareGridLevel (src/refinement/intrinsic3d.cpp:307-313)
 *   k_upsample                       SDFAlgorithms::upsample<VoxelSBR> + interpolate<VoxelSBR> (algorithms.cpp:118-235),
 *                                    called by Intrinsic3D::finishGridLevel (intrinsic3d.cpp:320-331)
 *   k_gather_voxels                  stream compaction of the surviving voxels (order preserved)
 *
 * After either operation the engine rebuilds its hash and neighbour tables on the device (rebuild_topology in i3d_engine.cu).
 * Iteration order of the result: pruning keeps the survivors in their previous order; upsampling emits the 8 children of
 * voxel i at 8 i + (4 z + 2 y + x), the reference's loop nest (its own order is that of a fresh std::unordered_map).
 */
#pragma once
#include "i3d_grid.cuh"

namespace i3d
{

// pass 1 (algorithms.cpp:373-396): valid in-shell voxels keep themselves and their existing +-x,+-y,+-z,+2x,+2y,+2z neighbours
__global__ void k_shell_keep(GridView g, double thres_shell, uint8_t* __restrict__ keep)
{
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (v >= g.n) return;
    if (!(g.weight[v] > 0.0f) || fabs(g.sdf[v]) > thres_shell) return;
    keep[v] = 1;
#pragma unroll
    for (int o = 0; o <= NB_Z2; ++o)
    {
        const int32_t nb = g.nbr[static_cast<int64_t>(o) * g.n + v];
        if (nb >= 0) keep[nb] = 1;          // benign race: every writer stores 1
    }
}

// pass 2 (:399-452): a voxel not kept by pass 1 survives iff some existing voxel of its 5x5x5 neighbourhood has the other sign
__global__ void k_shell_crossing(GridView g, const unsigned long long* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask,
                                 uint8_t* __restrict__ keep)
{
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (v >= g.n || keep[v]) return;
    const bool negative = g.sdf[v] < 0.0;
    const int X = g.x[v], Y = g.y[v], Z = g.z[v];
    bool crossing = false;
    for (int dz = -2; dz <= 2 && !crossing; ++dz)
        for (int dy = -2; dy <= 2 && !crossing; ++dy)
            for (int dx = -2; dx <= 2; ++dx)
            {
                if (dx == 0 && dy == 0 && dz == 0) continue;
                const int32_t nb = hash_find(keys, vals, mask, X + dx, Y + dy, Z + dz);
                if (nb < 0) continue;
                const bool nb_negative = g.sdf[nb] < 0.0;
                if (nb_negative != negative) { crossing = true; break; }
            }
    if (crossing) keep[v] = 2;               // distinct value: pass 2 must not feed back into other threads' pass-1 test
}

__global__ void k_gather_voxels(int64_t m, const int32_t* __restrict__ list, GridView g, VoxelArrays out)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= m) return;
    const int32_t v = list[i];
    out.x[i] = g.x[v]; out.y[i] = g.y[v]; out.z[i] = g.z[v];
    out.sdf0[i] = g.sdf0[v]; out.sdf[i] = g.sdf[v]; out.albedo[i] = g.albedo[v];
    out.weight[i] = g.weight[v]; out.rgb[i] = g.rgb[v];
}

__global__ void k_interleave_xyz(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z, int32_t* __restrict__ xyz)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    xyz[3 * i] = x[i]; xyz[3 * i + 1] = y[i]; xyz[3 * i + 2] = z[i];
}

// One thread per child voxel.  interpolate<VoxelSBR> (algorithms.cpp:118-197): float accumulation over the VALID corners of the
// parent's unit cube in math::interpolationWeights' corner order; a corner counts towards cnt_valid even when its weight is 0;
// weight := 0 when at most 4 corners are valid; colour rounded, everything else float -> double.
__global__ void __launch_bounds__(kThreads) k_upsample(GridView g, const unsigned long long* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask,
                                                       VoxelArrays out)
{
    const int64_t c = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (c >= 8 * g.n) return;
    const int64_t v = c >> 3;
    const int bx = static_cast<int>(c & 1), by = static_cast<int>((c >> 1) & 1), bz = static_cast<int>((c >> 2) & 1);
    const int X = g.x[v], Y = g.y[v], Z = g.z[v];
    // pos = p + 0.5 * (bx, by, bz): floor(pos) = p, fractional part 0 or 0.5
    const float t[3] = {bx ? 0.5f : 0.0f, by ? 0.5f : 0.0f, bz ? 0.5f : 0.0f};
    const int corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {1, 1, 0}, {0, 1, 1}, {1, 0, 1}, {1, 1, 1}};
    int32_t idx[8];
    idx[0] = static_cast<int32_t>(v);
    idx[1] = g.nbr[NB_XP * g.n + v]; idx[2] = g.nbr[NB_YP * g.n + v]; idx[3] = g.nbr[NB_ZP * g.n + v];
    idx[4] = g.nbr[NB_XY * g.n + v]; idx[5] = g.nbr[NB_YZ * g.n + v]; idx[6] = g.nbr[NB_XZ * g.n + v];
    idx[7] = hash_find(keys, vals, mask, X + 1, Y + 1, Z + 1);
    float a_sdf = 0.0f, a_w = 0.0f, a_alb = 0.0f, a_ref = 0.0f, a_c[3] = {0.0f, 0.0f, 0.0f}, sum_w = 0.0f;
    int cnt_valid = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k)
    {
        const int32_t nb = idx[k];
        if (nb < 0 || !(g.weight[nb] > 0.0f)) continue;            // grid->valid(coords[i])
        const float wx = corner[k][0] ? t[0] : FS(1.0f, t[0]);
        const float wy = corner[k][1] ? t[1] : FS(1.0f, t[1]);
        const float wz = corner[k][2] ? t[2] : FS(1.0f, t[2]);
        const float w = FM(FM(wx, wy), wz);
        const uchar4 col = g.rgb[nb];
        a_sdf = FA(a_sdf, FM(w, static_cast<float>(g.sdf0[nb])));
        a_c[0] = FA(a_c[0], FM(w, static_cast<float>(col.x)));
        a_c[1] = FA(a_c[1], FM(w, static_cast<float>(col.y)));
        a_c[2] = FA(a_c[2], FM(w, static_cast<float>(col.z)));
        a_w = FA(a_w, FM(w, g.weight[nb]));
        a_alb = FA(a_alb, FM(w, static_cast<float>(g.albedo[nb])));
        a_ref = FA(a_ref, FM(w, static_cast<float>(g.sdf[nb])));
        sum_w = FA(sum_w, w);
        ++cnt_valid;
    }
    if (sum_w > 0.0f)
    {
        a_sdf = FD(a_sdf, sum_w); a_w = FD(a_w, sum_w); a_alb = FD(a_alb, sum_w); a_ref = FD(a_ref, sum_w);
        a_c[0] = FD(a_c[0], sum_w); a_c[1] = FD(a_c[1], sum_w); a_c[2] = FD(a_c[2], sum_w);
    }
    if (cnt_valid <= 4) a_w = 0.0f;
    out.x[c] = 2 * X + bx; out.y[c] = 2 * Y + by; out.z[c] = 2 * Z + bz;
    out.sdf0[c] = static_cast<double>(a_sdf);
    out.sdf[c] = static_cast<double>(a_ref);
    out.albedo[c] = static_cast<double>(a_alb);
    out.weight[c] = fmaxf(a_w, 0.0f);
    // round(avg_color).cast<unsigned char>() with nv::round(Vec3f) = (v + 0.5f).cast<int>() (include/nv/mat.h:90); values are in [0, 255]
    out.rgb[c] = make_uchar4(static_cast<unsigned char>(__float2int_rz(FA(a_c[0], 0.5f))), static_cast<unsigned char>(__float2int_rz(FA(a_c[1], 0.5f))),
                             static_cast<unsigned char>(__float2int_rz(FA(a_c[2], 0.5f))), 0);
}

} // namespace i3d
