/*
 * i3d_grid.cuh — what every device module of the engine shares about the grid: the neighbour-table slots, the block size, the device
 * hash (coordinates -> voxel index), the explicitly rounded float operations, the grid view with the per-voxel operators both modules
 * evaluate (surface normal, intensity), the voxel arrays a new voxel set is written into, the normal rule of a depth plane (fusion and
 * tracking) and the subvolume table and SH blend of the lighting.  No kernels: i3d_kernels.cuh, i3d_observe.cuh, i3d_lighting.cuh and
 * i3d_gridops.cuh (the engine's module), i3d_fusion.cuh (the fusion's), i3d_frames.cuh (the frames'), i3d_mesh.cuh / i3d_vis.cuh (the
 * surface extraction's) and i3d_render.cuh / i3d_track.cuh (the renderer's) all include it.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace i3d
{

// neighbour-table slots
enum { NB_XP = 0, NB_XM, NB_YP, NB_YM, NB_ZP, NB_ZM, NB_X2, NB_Y2, NB_Z2, NB_XY, NB_XZ, NB_YZ, NB_COUNT };

constexpr int kThreads = 256;

// ----------------------------------------------------------------------------------------------
// exact float arithmetic (no FMA contraction): must round like oracle.cpp / the reference's float code
// ----------------------------------------------------------------------------------------------
#define FM(a, b) __fmul_rn((a), (b))
#define FA(a, b) __fadd_rn((a), (b))
#define FS(a, b) __fsub_rn((a), (b))
#define FD(a, b) __fdiv_rn((a), (b))

// ----------------------------------------------------------------------------------------------
// device hash table of the grid (replaces unordered_map::find, sparse_voxel_grid.cpp:166-259)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t pack_key(int x, int y, int z)
{
    return ((static_cast<uint64_t>(x + (1 << 20)) & 0x1FFFFFull) << 42) | ((static_cast<uint64_t>(y + (1 << 20)) & 0x1FFFFFull) << 21) |
           (static_cast<uint64_t>(z + (1 << 20)) & 0x1FFFFFull);
}
__device__ __forceinline__ uint64_t mix64(uint64_t k)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return k;
}
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

// (noinline: runs once per grid upload; keeps the 12 probe loops out of the caller.  inline: one definition per translation unit)
inline __device__ __noinline__ int32_t hash_find(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask, int x, int y, int z)
{
    const unsigned long long key = pack_key(x, y, z);
    uint64_t slot = mix64(key) & mask;
    while (true)
    {
        const unsigned long long k = keys[slot];
        if (k == key) return vals[slot];
        if (k == kEmptyKey) return -1;
        slot = (slot + 1) & mask;
    }
}

// ----------------------------------------------------------------------------------------------
// the engine's grid as the per-voxel operators read it
// ----------------------------------------------------------------------------------------------
struct GridView
{
    int64_t n;
    const int32_t* x; const int32_t* y; const int32_t* z;
    const double* sdf0; const double* sdf; const double* albedo;
    const float* weight;
    const uchar4* rgb;
    const int32_t* nbr;    // [12][n]
    const double* sh;      // [9][n]
    float voxel_size, truncation;
};

// the voxel arrays a new voxel set is written into (grid-level transitions, fusion)
struct VoxelArrays
{
    int32_t* x; int32_t* y; int32_t* z;
    double* sdf0; double* sdf; double* albedo;
    float* weight;
    uchar4* rgb;
};

// SDFOperators::computeSurfaceNormal (src/sdf/operators.cpp:58-77): float forward differences.
__device__ __forceinline__ bool surface_normal_f(const GridView& g, int64_t v, float nrm[3])
{
    nrm[0] = nrm[1] = nrm[2] = 0.0f;
    const int32_t ix = g.nbr[NB_XP * g.n + v], iy = g.nbr[NB_YP * g.n + v], iz = g.nbr[NB_ZP * g.n + v];
    if (!(g.weight[v] > 0.0f) || ix < 0 || iy < 0 || iz < 0) return false;
    if (!(g.weight[ix] > 0.0f) || !(g.weight[iy] > 0.0f) || !(g.weight[iz] > 0.0f)) return false;
    const float s0 = static_cast<float>(g.sdf[v]);
    float g0 = FS(static_cast<float>(g.sdf[ix]), s0);
    float g1 = FS(static_cast<float>(g.sdf[iy]), s0);
    float g2 = FS(static_cast<float>(g.sdf[iz]), s0);
    const float sq = FA(FA(FM(g0, g0), FM(g1, g1)), FM(g2, g2));
    const float len = __fsqrt_rn(sq);
    if (len != 0.0f) { g0 = FD(g0, len); g1 = FD(g1, len); g2 = FD(g2, len); }
    nrm[0] = g0; nrm[1] = g1; nrm[2] = g2;
    return !(g0 == 0.0f && g1 == 0.0f && g2 == 0.0f);
}

// ----------------------------------------------------------------------------------------------
// normals of a depth plane (k_fuse_normals, k_track_normals)
// ----------------------------------------------------------------------------------------------
// computeNormals(vertex_map, 0.3) (processing.cpp:72-118) at pixel i of a W x H depth plane, with the vertex map evaluated on the fly as
// computeVertexMap (:49-69) builds it: (x0 d, y0 d, d), x0 = (x - cx) * (1 / fx).  Central tangents, n = (t_y x t_x).normalized(); zero
// where undefined.
__device__ __forceinline__ float3 depth_normal(const float* __restrict__ depth, int W, int H, float fx, float fy, float cx, float cy, int64_t i)
{
    const int y = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<int64_t>(y) * W);
    float n[3] = {0.0f, 0.0f, 0.0f};
    if (x >= 1 && y >= 1 && x < W - 1 && y < H - 1 && depth[i] != 0.0f)
    {
        const float fxi = FD(1.0f, fx), fyi = FD(1.0f, fy);
        auto vertex = [&](int u, int v, float out[3]) {
            const float d = depth[static_cast<int64_t>(v) * W + u];
            out[0] = FM(FM(FS(static_cast<float>(u), cx), fxi), d);
            out[1] = FM(FM(FS(static_cast<float>(v), cy), fyi), d);
            out[2] = d;
        };
        float vx0[3], vx1[3], vy0[3], vy1[3];
        vertex(x - 1, y, vx0);
        vertex(x + 1, y, vx1);
        vertex(x, y - 1, vy0);
        vertex(x, y + 1, vy1);
        if (vx0[2] != 0.0f && vx1[2] != 0.0f && vy0[2] != 0.0f && vy1[2] != 0.0f)
        {
            const float tx[3] = {FS(vx1[0], vx0[0]), FS(vx1[1], vx0[1]), FS(vx1[2], vx0[2])};
            const float ty[3] = {FS(vy1[0], vy0[0]), FS(vy1[1], vy0[1]), FS(vy1[2], vy0[2])};
            const float lx = __fsqrt_rn(FA(FA(FM(tx[0], tx[0]), FM(tx[1], tx[1])), FM(tx[2], tx[2])));
            const float ly = __fsqrt_rn(FA(FA(FM(ty[0], ty[0]), FM(ty[1], ty[1])), FM(ty[2], ty[2])));
            if (lx < 0.3f && ly < 0.3f)
            {
                float c[3] = {FS(FM(ty[1], tx[2]), FM(ty[2], tx[1])), FS(FM(ty[2], tx[0]), FM(ty[0], tx[2])), FS(FM(ty[0], tx[1]), FM(ty[1], tx[0]))};
                const float sq = FA(FA(FM(c[0], c[0]), FM(c[1], c[1])), FM(c[2], c[2]));
                if (sq > 0.0f) { const float l = __fsqrt_rn(sq); c[0] = FD(c[0], l); c[1] = FD(c[1], l); c[2] = FD(c[2], l); }
                n[0] = c[0]; n[1] = c[1]; n[2] = c[2];
            }
        }
    }
    return make_float3(n[0], n[1], n[2]);
}

// nv::intensity(unsigned char r, g, b) (src/color_util.cpp:41-46)
__device__ __forceinline__ float intensity_u8(uchar4 c) { return FA(FA(FM(0.299f, static_cast<float>(c.x)), FM(0.587f, static_cast<float>(c.y))), FM(0.114f, static_cast<float>(c.z))); }

// ----------------------------------------------------------------------------------------------
// subvolumes of the SVSH lighting (Subvolumes, src/lighting/subvolumes.cpp)
// ----------------------------------------------------------------------------------------------
struct SubvolGrid
{
    int lo[3];
    int dim[3];
    const int32_t* table;    // [dim z][dim y][dim x] -> subvolume id or -1
    float inv_size;          // 1.0f / size_ (Subvolumes::pointToIndexFloat, src/lighting/subvolumes.cpp:262-265)
    __host__ __device__ int64_t cells() const { return static_cast<int64_t>(dim[0]) * dim[1] * dim[2]; }
    __device__ __forceinline__ int find(int x, int y, int z) const
    {
        x -= lo[0]; y -= lo[1]; z -= lo[2];
        if (x < 0 || y < 0 || z < 0 || x >= dim[0] || y >= dim[1] || z >= dim[2]) return -1;
        return table[(static_cast<int64_t>(z) * dim[1] + y) * dim[0] + x];
    }
};

// Subvolumes::interpolate(linear) at voxelToWorld of voxel v (subvolumes.cpp:165-205, math::interpolationWeights / average, src/math.cpp:74-128),
// the blend of the SVSH lighting's per-voxel coefficients (k_svsh_interpolate) and of the shading colour modes (i3d_vis.cuh):
// float trilinear weights of the 8 surrounding subvolumes at p / size - 0.5, missing cubes and zero weights skipped, the sub_sh [S][9]
// vectors summed in double (product and sum rounded separately), times double(1.0f / sum of the weights).  avg must be zero on entry;
// it stays zero when no weight is left.
// The core takes the world point as coord(d), d = 0, 1, 2: svsh_blend_at the point p itself, svsh_blend voxel v's FM(float(c), voxel_size).
template <class Coord>
__device__ __forceinline__ void svsh_blend_core(Coord&& coord, const SubvolGrid& sg, const double* __restrict__ sub_sh, double (&avg)[9])
{
    int v0[3]; float wg[3];
#pragma unroll
    for (int d = 0; d < 3; ++d)
    {
        const float pos = FS(FM(coord(d), sg.inv_size), 0.5f);     // pointToIndexCoord
        const float fl = floorf(pos);
        v0[d] = static_cast<int>(fl);
        wg[d] = FS(pos, fl);
    }
    // math::interpolationWeights corner order (src/math.cpp:103-128)
    const int corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {1, 1, 0}, {0, 1, 1}, {1, 0, 1}, {1, 1, 1}};
    float sum_w = 0.0f;
#pragma unroll
    for (int i = 0; i < 8; ++i)
    {
        const float wx = corner[i][0] ? wg[0] : FS(1.0f, wg[0]);
        const float wy = corner[i][1] ? wg[1] : FS(1.0f, wg[1]);
        const float wz = corner[i][2] ? wg[2] : FS(1.0f, wg[2]);
        const float w = FM(FM(wx, wy), wz);
        const int id = sg.find(v0[0] + corner[i][0], v0[1] + corner[i][1], v0[2] + corner[i][2]);
        if (id < 0 || w == 0.0f) continue;
        const double wd = static_cast<double>(w);
        const double* src = sub_sh + static_cast<int64_t>(id) * 9;
#pragma unroll
        for (int k = 0; k < 9; ++k) avg[k] = (sum_w == 0.0f) ? wd * src[k] : avg[k] + wd * src[k];
        sum_w = FA(sum_w, w);
    }
    if (sum_w != 0.0f)
    {
        const double inv = static_cast<double>(FD(1.0f, sum_w));
#pragma unroll
        for (int k = 0; k < 9; ++k) avg[k] *= inv;
    }
}

__device__ __forceinline__ void svsh_blend(const GridView& g, int64_t v, const SubvolGrid& sg, const double* __restrict__ sub_sh, double (&avg)[9])
{
    const int c[3] = {g.x[v], g.y[v], g.z[v]};
    svsh_blend_core([&](int d) { return FM(static_cast<float>(c[d]), g.voxel_size); }, sg, sub_sh, avg);
}

__device__ __forceinline__ void svsh_blend_at(const float (&p)[3], const SubvolGrid& sg, const double* __restrict__ sub_sh, double (&avg)[9])
{
    svsh_blend_core([&](int d) { return p[d]; }, sg, sub_sh, avg);
}

// sh . basis(n) of Shading::computeShading on a unit normal: the basis in the order of Q9 computed in float, the dot product summed
// k = 0..8 left to right (vis_shading multiplies it by the albedo)
__device__ __forceinline__ float sh_dot(const float n[3], const float sh[9])
{
    const float x = n[0], y = n[1], z = n[2];
    const float b[9] = {1.0f, y, z, x, FM(x, y), FM(y, z), FA(FS(-FM(x, x), FM(y, y)), FM(2.0f, FM(z, z))), FM(x, z), FS(FM(x, x), FM(y, y))};
    float d = FM(sh[0], b[0]);
#pragma unroll
    for (int k = 1; k < 9; ++k) d = FA(d, FM(sh[k], b[k]));
    return d;
}

// A lighting of the texture decomposition and the relit raster (I3DShLighting): global = the nine floats sh; otherwise the subvolume SH
// sub_sh [S][9] of the last estimate on the table sg, taken as it is when S = 1 and blended at the point by svsh_blend_at otherwise, then
// rounded to float
struct ShLight
{
    int global;
    float sh[9];
    SubvolGrid sg;
    const double* sub_sh;
    int S;
};

__device__ __forceinline__ void sh_light_at(const ShLight& L, const float (&p)[3], float (&sh)[9])
{
    if (L.global)
    {
#pragma unroll
        for (int k = 0; k < 9; ++k) sh[k] = L.sh[k];
        return;
    }
    double avg[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) avg[k] = L.S == 1 ? L.sub_sh[k] : 0.0;
    if (L.S != 1) svsh_blend_at(p, L.sg, L.sub_sh, avg);
#pragma unroll
    for (int k = 0; k < 9; ++k) sh[k] = __double2float_rn(avg[k]);
}

} // namespace i3d
