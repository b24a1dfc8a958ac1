/*
 * i3d_distance.cuh — the distance between the resident mesh and a reference mesh (DESIGN.md §6u): area-uniform samples of one mesh, the
 * nearest face of the other through a uniform search grid, and per-direction statistics summed in a fixed order.  Restated in numpy
 * float32 by tests/distance_ref.py.  FM / FA / FS / FD are one IEEE float operation each (no contraction).
 *
 * Samples.  Face (v0, v1, v2) is split into L^2 congruent sub-triangles; sample s in [0, L^2) is the centroid of one of them:
 *   s <  L(L+1)/2: "up" (i, j), i + j <= L - 1, rows i ascending, j ascending in a row; (a, b) = (FD(FA(i, 1/3), L), FD(FA(j, 1/3), L))
 *   s >= L(L+1)/2: "down" (i, j), i + j <= L - 2, same order from s - L(L+1)/2;       (a, b) with 2/3 in place of 1/3
 *   1/3 = FD(1, 3), 2/3 = FD(2, 3); w0 = FS(FS(1, a), b); P = FA(FA(FM(w0, v0), FM(a, v1)), FM(b, v2)) per coordinate.
 *   area = FM(1/2, sqrt(FA(FA(FM(n0, n0), FM(n1, n1)), FM(n2, n2)))) (__fsqrt_rn), n = (v1 - v0) x (v2 - v0), each component
 *   FS(FM(e1[p], e2[q]), FM(e1[q], e2[p])); the sample's weight is double(area) / double(L^2).  Samples are never stored.
 *
 * The closest point and the nearest-face query are in i3d_distance_query.cuh, which the mesh-to-grid conversion shares.
 *
 * Closest point (dist_point_tri_d2): Ericson, Real-Time Collision Detection §5.1.5, in the order written below, then d^2 = dot(p - q,
 * p - q), dot(x, y) = FA(FA(FM(x0, y0), FM(x1, y1)), FM(x2, y2)).  A triangle with dot(n, n) = 0, one where a division of the
 * procedure would have a denominator that is not > 0 and one whose interior (v, w) fall outside v, w >= 0, FA(v, w) <= 1 is measured
 * as its three edges instead: the smallest d^2 to the segments ab, bc, ca (t = FD(dot(p - s0, s1 - s0), dot(s1 - s0, s1 - s0)) clamped
 * to [0, 1], 0 for a zero-length segment; q = FA(s0, FM(t, s1 - s0))).  For a sliver (kDistSliver) d^2 is fminf(procedure, edges).
 *
 * Nearest face: the lexicographic minimum of (d^2, face id) over every face with d^2 <= FM(max_distance, max_distance).  No such face:
 * unmatched (d^2 = +inf, face -1).  The grid cannot change the result, only which faces are tested:
 *   cell_of(x) = floor(clamp(FD(FS(x, lo), h), 0, n - 1)) per axis, lo = FS(bbox min, max_distance) of the target's faces, h the cell edge.
 *   A face is listed in every cell of cell_of(its float AABB); cell_of is monotone, so each point of the face lies in a listed cell.
 *   The query visits the Chebyshev shells r = 0, 1, ... of cells around cell_of(p) (clamped, so points outside the box work).  After
 *   shell r, every unvisited face lies beyond one of the block's faces that still has cells behind it; lb is p's distance to the
 *   nearest such plane, in double, less a margin of 2^-16 (|lo|, |hi|, extent, h and |p| maxima) that covers the float rounding of
 *   cell_of and of d^2 many times over.  The search stops when no such plane is left or lb > 0 and lb^2 > the current best d^2 (or
 *   max_distance^2 while unmatched), so an equal d^2 in a later shell is never skipped.
 *
 * Statistics: one thread per sample; per block a fixed shuffle tree per warp and the warps in order (dist_block_reduce), then
 * k_dist_finish sums the blocks in order.  No atomics: every number is bit-identical from run to run.
 */
#pragma once
#include "i3d_distance_query.cuh"

namespace i3d
{

// Stat slots of one direction: 0 matched area, 1 matched samples, 2 area, 3 unmatched area, 4 sum w d, 5 sum w d^2, 6 max d (a
// maximum, not a sum), 7 point-triangle tests, 8 + t area with d^2 <= tau_t^2
constexpr int kDistStats = 16;
constexpr unsigned kDistStatsMax = 1u << 6;
// Bounds slots of a target mesh: -min x, y, z and max x, y, z of its faces (maxima), the sum of its edge lengths
constexpr int kDistBounds = 7;
constexpr unsigned kDistBoundsMax = 0x3Fu;

struct DistQuery
{
    float max_distance; int L; int num_thresholds;
    float tau[I3D_DISTANCE_MAX_THRESHOLDS];
};

// Sample s of face f of m: the point P and the face's float area
__device__ __forceinline__ void dist_sample(const DistMesh& m, int64_t f, int s, int L, float* P, float& area)
{
    const int3 fv = m.faces[f];
    const float* p0 = m.vpos + 3 * static_cast<size_t>(fv.x);
    const float* p1 = m.vpos + 3 * static_cast<size_t>(fv.y);
    const float* p2 = m.vpos + 3 * static_cast<size_t>(fv.z);
    const int nup = L * (L + 1) / 2;
    const bool down = s >= nup;
    int r = down ? s - nup : s, row = down ? L - 1 : L, i = 0;
    while (r >= row) { r -= row; --row; ++i; }
    const float off = down ? FD(2.0f, 3.0f) : FD(1.0f, 3.0f);
    const float a = FD(FA(static_cast<float>(i), off), static_cast<float>(L)), b = FD(FA(static_cast<float>(r), off), static_cast<float>(L));
    const float w0 = FS(FS(1.0f, a), b);
    float e1[3], e2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        P[k] = FA(FA(FM(w0, p0[k]), FM(a, p1[k])), FM(b, p2[k]));
        e1[k] = FS(p1[k], p0[k]); e2[k] = FS(p2[k], p0[k]);
    }
    const float n0 = FS(FM(e1[1], e2[2]), FM(e1[2], e2[1]));
    const float n1 = FS(FM(e1[2], e2[0]), FM(e1[0], e2[2]));
    const float n2 = FS(FM(e1[0], e2[1]), FM(e1[1], e2[0]));
    area = FM(0.5f, __fsqrt_rn(FA(FA(FM(n0, n0), FM(n1, n1)), FM(n2, n2))));
}

// Block reduction of NS slots into out[blockIdx.x][NS]: per warp a shuffle-down tree, then the warps in order; slot j is a maximum when
// bit j of max_mask is set, else a sum.  Every thread of the block calls it.
template <int NS>
__device__ __forceinline__ void dist_block_reduce(double* v, unsigned max_mask, double* __restrict__ out)
{
    __shared__ double s[kThreads / 32][NS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < NS; ++j)
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
        {
            const double t = __shfl_down_sync(0xffffffffu, v[j], o);
            v[j] = ((max_mask >> j) & 1u) ? fmax(v[j], t) : v[j] + t;
        }
    }
    if (lane == 0)
    {
#pragma unroll
        for (int j = 0; j < NS; ++j) s[warp][j] = v[j];
    }
    __syncthreads();
    if (threadIdx.x < NS)
    {
        const int j = threadIdx.x;
        const bool mx = (max_mask >> j) & 1u;
        double t = s[0][j];
        for (int w = 1; w < kThreads / 32; ++w) t = mx ? fmax(t, s[w][j]) : t + s[w][j];
        out[static_cast<size_t>(blockIdx.x) * NS + j] = t;
    }
}

// Per block: the faces' AABB (kDistBounds slots, minima negated) and the sum of their float edge lengths
__global__ void __launch_bounds__(kThreads) k_dist_bounds(DistMesh m, double* __restrict__ partials)
{
    const int64_t f = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    double v[kDistBounds];
#pragma unroll
    for (int j = 0; j < 6; ++j) v[j] = -1e300;
    v[6] = 0.0;
    if (f < m.F)
    {
        const int3 fv = m.faces[f];
        const float* p[3] = {m.vpos + 3 * static_cast<size_t>(fv.x), m.vpos + 3 * static_cast<size_t>(fv.y), m.vpos + 3 * static_cast<size_t>(fv.z)};
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            v[k] = -static_cast<double>(fminf(fminf(p[0][k], p[1][k]), p[2][k]));
            v[3 + k] = static_cast<double>(fmaxf(fmaxf(p[0][k], p[1][k]), p[2][k]));
        }
        double len = 0.0;
#pragma unroll
        for (int q = 0; q < 3; ++q)
        {
            float e[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) e[k] = FS(p[(q + 1) % 3][k], p[q][k]);
            len += static_cast<double>(__fsqrt_rn(dist_dot(e, e)));
        }
        v[6] = len;
    }
    dist_block_reduce<kDistBounds>(v, kDistBoundsMax, partials);
}

// The cell range of face f's float AABB
__device__ __forceinline__ void dist_face_cells(const DistMesh& m, const DistGrid& g, int64_t f, int* c0, int* c1)
{
    const int3 fv = m.faces[f];
    const float* p0 = m.vpos + 3 * static_cast<size_t>(fv.x);
    const float* p1 = m.vpos + 3 * static_cast<size_t>(fv.y);
    const float* p2 = m.vpos + 3 * static_cast<size_t>(fv.z);
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        c0[k] = dist_cell(fminf(fminf(p0[k], p1[k]), p2[k]), g.lo[k], g.h, g.n[k]);
        c1[k] = dist_cell(fmaxf(fmaxf(p0[k], p1[k]), p2[k]), g.lo[k], g.h, g.n[k]);
    }
}

// Sum over faces of the cells their AABB covers (integer atomics: the total does not depend on their order)
__global__ void __launch_bounds__(kThreads) k_dist_entries(DistMesh m, DistGrid g, unsigned long long* __restrict__ total)
{
    const int64_t f = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    unsigned long long n = 0;
    if (f < m.F)
    {
        int c0[3], c1[3];
        dist_face_cells(m, g, f, c0, c1);
        n = static_cast<unsigned long long>(c1[0] - c0[0] + 1) * (c1[1] - c0[1] + 1) * (c1[2] - c0[2] + 1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(total, n);
}

// Count (off == nullptr) or fill: per face, every cell of its AABB.  The fill's order inside a cell does not matter (see the top).
__global__ void __launch_bounds__(kThreads) k_dist_insert(DistMesh m, DistGrid g, const int64_t* __restrict__ off, int32_t* __restrict__ cnt,
                                                          int32_t* __restrict__ list)
{
    const int64_t f = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (f >= m.F) return;
    int c0[3], c1[3];
    dist_face_cells(m, g, f, c0, c1);
    for (int z = c0[2]; z <= c1[2]; ++z)
        for (int y = c0[1]; y <= c1[1]; ++y)
            for (int x = c0[0]; x <= c1[0]; ++x)
            {
                const int64_t cell = (static_cast<int64_t>(z) * g.n[1] + y) * g.n[0] + x;
                const int slot = atomicAdd(cnt + cell, 1);
                if (off) list[off[cell] + slot] = static_cast<int32_t>(f);
            }
}

// The query kernels are bounded to two blocks of kThreads per SM: the register limit of three blocks (80) spills.
// One thread per sample of src against tgt: stat partials per block, and the per-sample (d^2, face) when keep_d2 is set
__global__ void __launch_bounds__(kThreads, 2) k_dist_samples(DistMesh src, DistMesh tgt, DistGrid g, DistQuery q, float* __restrict__ keep_d2,
                                                           int32_t* __restrict__ keep_face, double* __restrict__ partials)
{
    const int LL = q.L * q.L;
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const bool live = t < src.F * LL;
    float area = 0.0f, bd2 = 0.0f; int bf = -1; long long tests = 0;
    if (live)
    {
        const int64_t f = t / LL;
        float P[3];
        dist_sample(src, f, static_cast<int>(t - f * LL), q.L, P, area);
        dist_nearest(P, tgt, g, FM(q.max_distance, q.max_distance), bd2, bf, tests);
        if (keep_d2) { keep_d2[t] = bd2; keep_face[t] = bf; }
    }
    // the slots are formed after the search, so that they are not live across it
    double v[kDistStats];
#pragma unroll
    for (int j = 0; j < kDistStats; ++j) v[j] = 0.0;
    if (live)
    {
        const double w = __ddiv_rn(static_cast<double>(area), static_cast<double>(LL));
        v[2] = w;
        v[7] = static_cast<double>(tests);
        if (bf >= 0)
        {
            const double d = __dsqrt_rn(static_cast<double>(bd2));
            v[0] = w; v[1] = 1.0;
            v[4] = __dmul_rn(w, d); v[5] = __dmul_rn(w, static_cast<double>(bd2)); v[6] = d;
#pragma unroll
            for (int k = 0; k < I3D_DISTANCE_MAX_THRESHOLDS; ++k)
                if (k < q.num_thresholds && bd2 <= FM(q.tau[k], q.tau[k])) v[8 + k] = w;
        }
        else v[3] = w;
    }
    dist_block_reduce<kDistStats>(v, kDistStatsMax, partials);
}

// One warp per slot: lane l takes blocks l, l + 32, ... in order, then a fixed shuffle tree
__global__ void k_dist_finish(int blocks, const double* __restrict__ partials, double* __restrict__ stats)
{
    const int j = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (j >= kDistStats) return;
    const bool mx = (kDistStatsMax >> j) & 1u;
    double s = 0.0;
    for (int b = lane; b < blocks; b += 32) s = mx ? fmax(s, partials[static_cast<size_t>(b) * kDistStats + j]) : s + partials[static_cast<size_t>(b) * kDistStats + j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
    {
        const double t = __shfl_down_sync(0xffffffffu, s, o);
        s = mx ? fmax(s, t) : s + t;
    }
    if (lane == 0) stats[j] = s;
}

// One thread per vertex of src: its distance (sqrt of d^2, +inf unmatched) and face; the point-triangle tests summed per warp
__global__ void __launch_bounds__(kThreads, 2) k_dist_vertices(DistMesh src, DistMesh tgt, DistGrid g, float max_distance, float* __restrict__ vdist,
                                                            int32_t* __restrict__ vface, unsigned long long* __restrict__ tests_total)
{
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    long long tests = 0;
    if (t < src.V)
    {
        const float* p = src.vpos + 3 * static_cast<size_t>(t);
        const float P[3] = {p[0], p[1], p[2]};
        float bd2; int bf;
        dist_nearest(P, tgt, g, FM(max_distance, max_distance), bd2, bf, tests);
        vdist[t] = bf >= 0 ? __fsqrt_rn(bd2) : bd2;
        vface[t] = bf;
    }
    unsigned long long n = static_cast<unsigned long long>(tests);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(tests_total, n);
}

} // namespace i3d
