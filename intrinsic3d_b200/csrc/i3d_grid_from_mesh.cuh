/*
 * i3d_grid_from_mesh.cuh — the voxel grid from a triangle mesh (DESIGN.md §6v): the narrow-band signed distance on the lattice
 * c * voxel_size, signed by angle-weighted pseudonormals (Baerentzen & Aanaes 2005).  Restated in numpy by tests/grid_from_mesh_ref.py.
 *
 * Distance.  p = FM(float(c), voxel_size) per axis; b = FM(band, voxel_size); the nearest face is dist_nearest with lim2 = FM(b, b)
 * (i3d_distance_query.cuh).  No face within the band: the voxel is not emitted.  The feature of the closest point and p - q come from
 * dist_point_tri on that face, the same arithmetic as the distance.  |sdf| = double(__fsqrt_rn(d^2)).
 *
 * Topology.  Vertices are welded by exact float position (-0 as +0): the representative of a position is its lowest vertex index.
 * Edges are keyed by the welded pair.  In double, every operation explicit (no DFMA): a face's unit normal n / sqrt(n . n), n = (b - a)
 * x (c - a) of the float positions widened; dot(n, n) = 0 makes the face degenerate, and a degenerate face contributes nothing.  The
 * corner angle at vertex k is atan2(|u x w|, u . w), u, w the edges from it.  Sums run over the incidences in ascending face id (stable
 * radix sorts of 3 f + k by welded vertex and by welded edge; one thread per run), starting from 0:
 *   vertex pseudonormal = sum of angle * unit normal, edge pseudonormal = sum of unit normals, interior: the face's unit normal.
 * An edge is on the boundary when exactly one non-degenerate face uses it; a vertex when a boundary edge ends at it.
 *
 * Sign.  d = p - q (float, widened), dot = d . N, dd = d . d, nn = N . N in double, left to right.  d^2 = 0: sdf = +0.  Else nn = 0 or
 * dot = 0: dropped; a boundary feature with dot * dot < (I3D_GRID_FROM_MESH_RIM_COS^2 dd) nn: dropped; else sdf = +-|sdf| by the sign
 * of dot.
 *
 * Candidates.  Brick B (voxels 8 B + l, l in [0, 8)^3) is a candidate when dist_point_tri_d2(FM(FA(8 B, 3.5), voxel_size), face) <=
 * r2 for a face whose AABB grown by b covers it, r = b + 3.5 sqrt(3) voxel_size + voxel_size: every voxel within b of a face lies in
 * such a brick.  The candidates only decide which voxels are queried, never a result.  The bricks are sorted by the brick part of
 * fuse_order_key and each brick's voxels queried in (lz, ly, lx) order, so the kept voxels come out in canonical 8^3-brick-major order.
 */
#pragma once
#include "i3d_distance_query.cuh"

namespace i3d
{

// counter slots
enum { GFM_BEYOND = 0, GFM_RIM, GFM_ZERO_NORMAL, GFM_ZERO_DOT, GFM_NEGATIVE, GFM_TESTS, GFM_EMITTED, GFM_WELDED, GFM_BOUNDARY, GFM_FILL,
       GFM_PAIRS, GFM_COUNTERS };
constexpr int kGfmBrickBias = 1 << 17;           // brick coordinate + bias = (c + 2^20) >> 3 for c = 8 B + l

struct GfmConst
{
    float voxel_size, b, r2;
    double inv_voxel_size_d, b_d;
};

__device__ __forceinline__ uint32_t gfm_bits(float x) { return __float_as_uint(x == 0.0f ? 0.0f : x); }

__device__ __forceinline__ bool gfm_same_pos(const float* vpos, int32_t u, int32_t v)
{
    const float* a = vpos + 3 * static_cast<size_t>(u);
    const float* b = vpos + 3 * static_cast<size_t>(v);
    return gfm_bits(a[0]) == gfm_bits(b[0]) && gfm_bits(a[1]) == gfm_bits(b[1]) && gfm_bits(a[2]) == gfm_bits(b[2]);
}

// brick key: the brick part of fuse_order_key
__device__ __forceinline__ unsigned long long gfm_brick_key(int bx, int by, int bz)
{
    return (static_cast<unsigned long long>(bz + kGfmBrickBias) << 46) | (static_cast<unsigned long long>(by + kGfmBrickBias) << 28) |
           (static_cast<unsigned long long>(bx + kGfmBrickBias) << 10);
}

// the lattice coordinates of candidate voxel l in [0, 512) of brick key K
__device__ __forceinline__ void gfm_voxel(unsigned long long K, int l, int c[3])
{
    const int bx = static_cast<int>((K >> 10) & 0x3FFFFull), by = static_cast<int>((K >> 28) & 0x3FFFFull), bz = static_cast<int>(K >> 46);
    c[0] = ((bx << 3) | (l & 7)) - (1 << 20);
    c[1] = ((by << 3) | ((l >> 3) & 7)) - (1 << 20);
    c[2] = ((bz << 3) | (l >> 6)) - (1 << 20);
}

__device__ __forceinline__ void gfm_add(unsigned long long* counters, int slot, unsigned v)
{
    v = __reduce_add_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(counters + slot, static_cast<unsigned long long>(v));
}

__device__ __forceinline__ double gfm_dot(const double* x, const double* y) { return __dadd_rn(__dadd_rn(__dmul_rn(x[0], y[0]), __dmul_rn(x[1], y[1])), __dmul_rn(x[2], y[2])); }

__device__ __forceinline__ void gfm_cross(const double* u, const double* w, double* n)
{
    n[0] = __dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1]));
    n[1] = __dsub_rn(__dmul_rn(u[2], w[0]), __dmul_rn(u[0], w[2]));
    n[2] = __dsub_rn(__dmul_rn(u[0], w[1]), __dmul_rn(u[1], w[0]));
}

// the edges from corner k of face fv: u to corner k + 1, w to corner k + 2, widened
__device__ __forceinline__ void gfm_corner_edges(const float* vpos, int3 fv, int k, double* u, double* w)
{
    const int ids[3] = {fv.x, fv.y, fv.z};
    const float* a = vpos + 3 * static_cast<size_t>(ids[k]);
    const float* b = vpos + 3 * static_cast<size_t>(ids[(k + 1) % 3]);
    const float* c = vpos + 3 * static_cast<size_t>(ids[(k + 2) % 3]);
#pragma unroll
    for (int j = 0; j < 3; ++j)
    {
        u[j] = __dsub_rn(static_cast<double>(b[j]), static_cast<double>(a[j]));
        w[j] = __dsub_rn(static_cast<double>(c[j]), static_cast<double>(a[j]));
    }
}

// ---- welding --------------------------------------------------------------------------------------------------------------------
__global__ void k_gfm_weld_z(int64_t V, const float* __restrict__ vpos, uint32_t* __restrict__ key, int32_t* __restrict__ idx)
{
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (v >= V) return;
    key[v] = gfm_bits(vpos[3 * v + 2]);
    idx[v] = static_cast<int32_t>(v);
}

__global__ void k_gfm_weld_xy(int64_t V, const float* __restrict__ vpos, const int32_t* __restrict__ idx, unsigned long long* __restrict__ key)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= V) return;
    const float* p = vpos + 3 * static_cast<size_t>(idx[i]);
    key[i] = (static_cast<unsigned long long>(gfm_bits(p[0])) << 32) | gfm_bits(p[1]);
}

// order: vertices sorted by position, equal positions in ascending index; the first of each run is the representative
__global__ void k_gfm_weld_runs(int64_t V, const float* __restrict__ vpos, const int32_t* __restrict__ order, int32_t* __restrict__ weld,
                                unsigned long long* __restrict__ counters)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    bool head = false;
    if (i < V)
    {
        const int32_t v = order[i];
        head = i == 0 || !gfm_same_pos(vpos, order[i - 1], v);
        if (head)
            for (int64_t j = i; j < V && (j == i || gfm_same_pos(vpos, order[j], v)); ++j) weld[order[j]] = v;
    }
    gfm_add(counters, GFM_WELDED, head ? 1u : 0u);
}

// ---- pseudonormals --------------------------------------------------------------------------------------------------------------
__global__ void k_gfm_face_normals(DistMesh m, double* __restrict__ fn)
{
    const int64_t f = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (f >= m.F) return;
    double u[3], w[3], n[3];
    gfm_corner_edges(m.vpos, m.faces[f], 0, u, w);
    gfm_cross(u, w, n);
    const double nn = gfm_dot(n, n);
    const double len = nn > 0.0 ? __dsqrt_rn(nn) : 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) fn[3 * f + k] = nn > 0.0 ? __ddiv_rn(n[k], len) : 0.0;
}

// per incidence i = 3 f + k: the welded corner k and the welded edge (corner k, corner k + 1)
__global__ void k_gfm_incidences(DistMesh m, const int32_t* __restrict__ weld, uint32_t* __restrict__ vk, int32_t* __restrict__ vi,
                                 unsigned long long* __restrict__ ek, int32_t* __restrict__ ei)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= 3 * m.F) return;
    const int3 fv = m.faces[i / 3];
    const int ids[3] = {fv.x, fv.y, fv.z};
    const int k = static_cast<int>(i % 3);
    const uint32_t wa = static_cast<uint32_t>(weld[ids[k]]), wb = static_cast<uint32_t>(weld[ids[(k + 1) % 3]]);
    vk[i] = wa; vi[i] = static_cast<int32_t>(i);
    ek[i] = (static_cast<unsigned long long>(min(wa, wb)) << 32) | max(wa, wb);
    ei[i] = static_cast<int32_t>(i);
}

__device__ __forceinline__ bool gfm_degenerate(const double* __restrict__ fn, int64_t f) { return fn[3 * f] == 0.0 && fn[3 * f + 1] == 0.0 && fn[3 * f + 2] == 0.0; }

// one thread per run of equal welded vertices (incidences in ascending face id): the sum of angle * unit normal, written to every corner
__global__ void k_gfm_vertex_normals(DistMesh m, const uint32_t* __restrict__ key, const int32_t* __restrict__ inc, const double* __restrict__ fn,
                                     double* __restrict__ vn)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const int64_t n = 3 * m.F;
    if (i >= n || (i > 0 && key[i - 1] == key[i])) return;
    double acc[3] = {0.0, 0.0, 0.0};
    int64_t j = i;
    for (; j < n && key[j] == key[i]; ++j)
    {
        const int64_t f = inc[j] / 3;
        if (gfm_degenerate(fn, f)) continue;
        double u[3], w[3], x[3];
        gfm_corner_edges(m.vpos, m.faces[f], inc[j] % 3, u, w);
        gfm_cross(u, w, x);
        const double ang = atan2(__dsqrt_rn(gfm_dot(x, x)), gfm_dot(u, w));
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[k] = __dadd_rn(acc[k], __dmul_rn(ang, fn[3 * f + k]));
    }
    for (int64_t t = i; t < j; ++t)
#pragma unroll
        for (int k = 0; k < 3; ++k) vn[3 * static_cast<int64_t>(inc[t]) + k] = acc[k];
}

// one thread per run of equal welded edges: the sum of unit normals and the boundary flag, written to every edge slot; a boundary edge
// marks its two welded vertices
__global__ void k_gfm_edge_normals(int64_t F, const unsigned long long* __restrict__ key, const int32_t* __restrict__ inc, const double* __restrict__ fn,
                                   double* __restrict__ en, uint8_t* __restrict__ eb, uint8_t* __restrict__ vb, unsigned long long* __restrict__ counters)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const int64_t n = 3 * F;
    bool boundary = false;
    if (i < n && (i == 0 || key[i - 1] != key[i]))
    {
        double acc[3] = {0.0, 0.0, 0.0};
        int used = 0;
        int64_t j = i;
        for (; j < n && key[j] == key[i]; ++j)
        {
            const int64_t f = inc[j] / 3;
            if (gfm_degenerate(fn, f)) continue;
            ++used;
#pragma unroll
            for (int k = 0; k < 3; ++k) acc[k] = __dadd_rn(acc[k], fn[3 * f + k]);
        }
        boundary = used == 1;
        for (int64_t t = i; t < j; ++t)
        {
#pragma unroll
            for (int k = 0; k < 3; ++k) en[3 * static_cast<int64_t>(inc[t]) + k] = acc[k];
            eb[inc[t]] = boundary ? 1 : 0;
        }
        if (boundary) { vb[key[i] >> 32] = 1; vb[key[i] & 0xFFFFFFFFull] = 1; }
    }
    gfm_add(counters, GFM_BOUNDARY, boundary ? 1u : 0u);
}

// ---- candidate bricks -----------------------------------------------------------------------------------------------------------
// The brick range of face f's AABB grown by b (a superset: floor / ceil in double)
__device__ __forceinline__ void gfm_face_bricks(const DistMesh& m, const GfmConst& C, int64_t f, int* b0, int* b1)
{
    const int3 fv = m.faces[f];
    const float* p0 = m.vpos + 3 * static_cast<size_t>(fv.x);
    const float* p1 = m.vpos + 3 * static_cast<size_t>(fv.y);
    const float* p2 = m.vpos + 3 * static_cast<size_t>(fv.z);
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        const double lo = static_cast<double>(fminf(fminf(p0[k], p1[k]), p2[k])) - C.b_d;
        const double hi = static_cast<double>(fmaxf(fmaxf(p0[k], p1[k]), p2[k])) + C.b_d;
        b0[k] = static_cast<int>(floor(floor(lo * C.inv_voxel_size_d) / 8.0));
        b1[k] = static_cast<int>(floor(ceil(hi * C.inv_voxel_size_d) / 8.0));
    }
}

__global__ void k_gfm_brick_pairs(DistMesh m, GfmConst C, unsigned long long* __restrict__ counters)
{
    const int64_t f = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    unsigned long long n = 0;
    if (f < m.F)
    {
        int b0[3], b1[3];
        gfm_face_bricks(m, C, f, b0, b1);
        n = static_cast<unsigned long long>(b1[0] - b0[0] + 1) * (b1[1] - b0[1] + 1) * (b1[2] - b0[2] + 1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(counters + GFM_PAIRS, n);
}

// The keys of the bricks of face f's range whose centre is within r of the face, in any order (sorted and made unique afterwards)
__global__ void k_gfm_brick_fill(DistMesh m, GfmConst C, unsigned long long* __restrict__ keys, unsigned long long* __restrict__ counters)
{
    const int64_t f = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (f >= m.F) return;
    int b0[3], b1[3];
    gfm_face_bricks(m, C, f, b0, b1);
    const int3 fv = m.faces[f];
    const float* a = m.vpos + 3 * static_cast<size_t>(fv.x);
    const float* b = m.vpos + 3 * static_cast<size_t>(fv.y);
    const float* c = m.vpos + 3 * static_cast<size_t>(fv.z);
    for (int z = b0[2]; z <= b1[2]; ++z)
        for (int y = b0[1]; y <= b1[1]; ++y)
            for (int x = b0[0]; x <= b1[0]; ++x)
            {
                const float P[3] = {FM(FA(static_cast<float>(8 * x), 3.5f), C.voxel_size), FM(FA(static_cast<float>(8 * y), 3.5f), C.voxel_size),
                                    FM(FA(static_cast<float>(8 * z), 3.5f), C.voxel_size)};
                if (dist_point_tri_d2(P, a, b, c) <= C.r2) keys[atomicAdd(counters + GFM_FILL, 1ull)] = gfm_brick_key(x, y, z);
            }
}

// ---- the query --------------------------------------------------------------------------------------------------------------------
struct GfmTopology
{
    const double* fn; const double* vn; const double* en;
    const uint8_t* eb; const uint8_t* vb; const int32_t* weld;
};

// The query kept under two blocks of kThreads per SM, as the distance's (dist_nearest's register need)
// One thread per candidate voxel i (brick i / 512, voxel i % 512 in (lz, ly, lx) order): keep bit 1, sdf, face and feature
__global__ void __launch_bounds__(kThreads, 2) k_gfm_query(int64_t nc, const unsigned long long* __restrict__ bricks, DistMesh m, DistGrid g, GfmConst C,
                                                         GfmTopology T, uint8_t* __restrict__ keep, double* __restrict__ sdf, int32_t* __restrict__ face,
                                                         int8_t* __restrict__ feat, unsigned long long* __restrict__ counters)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    long long tests = 0;
    int reason = -1;              // GFM_BEYOND, GFM_RIM, GFM_ZERO_NORMAL, GFM_ZERO_DOT, or -1 kept
    bool negative = false;
    if (i < nc)
    {
        int c[3];
        gfm_voxel(bricks[i >> 9], static_cast<int>(i & 511), c);
        const float p[3] = {FM(static_cast<float>(c[0]), C.voxel_size), FM(static_cast<float>(c[1]), C.voxel_size), FM(static_cast<float>(c[2]), C.voxel_size)};
        float bd2; int bf;
        dist_nearest(p, m, g, FM(C.b, C.b), bd2, bf, tests);
        int fe = -1;
        double s = 0.0;
        if (bf < 0) reason = GFM_BEYOND;
        else
        {
            const int3 fv = m.faces[bf];
            const int ids[3] = {fv.x, fv.y, fv.z};
            float dv[3];
            dist_point_tri(p, m.vpos + 3 * static_cast<size_t>(fv.x), m.vpos + 3 * static_cast<size_t>(fv.y), m.vpos + 3 * static_cast<size_t>(fv.z), &fe, dv);
            if (bd2 > 0.0f)
            {
                const double* N;
                bool boundary = false;
                if (fe == DIST_INTERIOR) N = T.fn + 3 * static_cast<int64_t>(bf);
                else if (fe <= DIST_VERTEX_C)
                {
                    N = T.vn + 3 * (3 * static_cast<int64_t>(bf) + fe);
                    boundary = T.vb[T.weld[ids[fe]]] != 0;
                }
                else
                {
                    const int slot = fe == DIST_EDGE_AB ? 0 : (fe == DIST_EDGE_BC ? 1 : 2);
                    N = T.en + 3 * (3 * static_cast<int64_t>(bf) + slot);
                    boundary = T.eb[3 * static_cast<int64_t>(bf) + slot] != 0;
                }
                const double d[3] = {static_cast<double>(dv[0]), static_cast<double>(dv[1]), static_cast<double>(dv[2])};
                const double Nv[3] = {N[0], N[1], N[2]};
                const double dot = gfm_dot(d, Nv), dd = gfm_dot(d, d), nn = gfm_dot(Nv, Nv);
                if (nn == 0.0) reason = GFM_ZERO_NORMAL;
                else if (dot == 0.0) reason = GFM_ZERO_DOT;
                else if (boundary && __dmul_rn(dot, dot) < __dmul_rn(__dmul_rn(I3D_GRID_FROM_MESH_RIM_COS * I3D_GRID_FROM_MESH_RIM_COS, dd), nn)) reason = GFM_RIM;
                else
                {
                    const double r = static_cast<double>(__fsqrt_rn(bd2));
                    s = dot > 0.0 ? r : -r;
                    negative = dot < 0.0;
                }
            }
        }
        keep[i] = reason < 0 ? 1 : 0;
        sdf[i] = s; face[i] = bf; feat[i] = static_cast<int8_t>(fe);
    }
    const bool live = i < nc;
    gfm_add(counters, GFM_BEYOND, reason == GFM_BEYOND);
    gfm_add(counters, GFM_RIM, reason == GFM_RIM);
    gfm_add(counters, GFM_ZERO_NORMAL, reason == GFM_ZERO_NORMAL);
    gfm_add(counters, GFM_ZERO_DOT, reason == GFM_ZERO_DOT);
    gfm_add(counters, GFM_NEGATIVE, negative);
    gfm_add(counters, GFM_EMITTED, live && reason < 0);
    unsigned long long t = static_cast<unsigned long long>(tests);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(counters + GFM_TESTS, t);
}

// k_fuse_convert's voxel: sdf0 = sdf, albedo 0.6, weight 1, colour 0; voxel j of the result is candidate act[j]
__global__ void k_gfm_gather(int64_t m, const int32_t* __restrict__ act, const unsigned long long* __restrict__ bricks, const double* __restrict__ sdf,
                             const int32_t* __restrict__ face, const int8_t* __restrict__ feat, VoxelArrays out, int32_t* __restrict__ last_face,
                             int8_t* __restrict__ last_feat)
{
    const int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (j >= m) return;
    const int64_t i = act[j];
    int c[3];
    gfm_voxel(bricks[i >> 9], static_cast<int>(i & 511), c);
    out.x[j] = c[0]; out.y[j] = c[1]; out.z[j] = c[2];
    out.sdf0[j] = sdf[i]; out.sdf[j] = sdf[i]; out.albedo[j] = 0.6;
    out.weight[j] = 1.0f; out.rgb[j] = make_uchar4(0, 0, 0, 0);
    last_face[j] = face[i]; last_feat[j] = feat[i];
}

} // namespace i3d
