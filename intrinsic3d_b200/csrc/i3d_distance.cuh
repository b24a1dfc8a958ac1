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
#include "i3d_distance.h"
#include "i3d_grid.cuh"

namespace i3d
{

// Stat slots of one direction: 0 matched area, 1 matched samples, 2 area, 3 unmatched area, 4 sum w d, 5 sum w d^2, 6 max d (a
// maximum, not a sum), 7 point-triangle tests, 8 + t area with d^2 <= tau_t^2
constexpr int kDistStats = 16;
constexpr unsigned kDistStatsMax = 1u << 6;
// Bounds slots of a target mesh: -min x, y, z and max x, y, z of its faces (maxima), the sum of its edge lengths
constexpr int kDistBounds = 7;
constexpr unsigned kDistBoundsMax = 0x3Fu;

// The search grid of a target mesh; off / cnt / faces are null while it is being counted
struct DistGrid
{
    float lo[3]; float h; int n[3];
    double margin;
    const int64_t* off; const int32_t* cnt; const int32_t* faces;
};

// A triangle with dot(n, n) <= 2^-20 dot(ab, ab) dot(ac, ac) (an angle below about 1e-3 rad) is a sliver: the float signs of Ericson's
// region tests cancel there, so its d^2 is also bounded by its edges'
constexpr float kDistSliver = 9.5367431640625e-07f;

struct DistQuery
{
    float max_distance; int L; int num_thresholds;
    float tau[I3D_DISTANCE_MAX_THRESHOLDS];
};

__device__ __forceinline__ float dist_dot(const float* x, const float* y) { return FA(FA(FM(x[0], y[0]), FM(x[1], y[1])), FM(x[2], y[2])); }

__device__ __forceinline__ float dist_seg_d2(const float* p, const float* s0, const float* s1)
{
    float e[3], sp[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { e[k] = FS(s1[k], s0[k]); sp[k] = FS(p[k], s0[k]); }
    const float ll = dist_dot(e, e);
    float t = ll > 0.0f ? FD(dist_dot(sp, e), ll) : 0.0f;
    t = t < 0.0f ? 0.0f : (t > 1.0f ? 1.0f : t);
    float d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) d[k] = FS(p[k], FA(s0[k], FM(t, e[k])));
    return dist_dot(d, d);
}

// float d^2 from p to triangle (a, b, c) (the rule at the top of the file)
__device__ __forceinline__ float dist_point_tri_d2(const float* p, const float* a, const float* b, const float* c)
{
    float ab[3], ac[3], ap[3], bp[3], cp[3], bc[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        ab[k] = FS(b[k], a[k]); ac[k] = FS(c[k], a[k]); ap[k] = FS(p[k], a[k]);
        bp[k] = FS(p[k], b[k]); cp[k] = FS(p[k], c[k]); bc[k] = FS(c[k], b[k]);
    }
    const float n[3] = {FS(FM(ab[1], ac[2]), FM(ab[2], ac[1])), FS(FM(ab[2], ac[0]), FM(ab[0], ac[2])), FS(FM(ab[0], ac[1]), FM(ab[1], ac[0]))};
    // the closest point: region 0, 1, 2 the vertex a, b, c; 3, 4, 5 the point at s along ab, ac, bc; 6 the interior a + v ab + w ac
    int region = 0;
    float s = 0.0f, vi = 0.0f, wi = 0.0f;
    const float nn = dist_dot(n, n);
    bool edges = !(nn > 0.0f);
    const bool sliver = !(nn > FM(FM(kDistSliver, dist_dot(ab, ab)), dist_dot(ac, ac)));
    if (!edges)
    {
        const float d1 = dist_dot(ab, ap), d2 = dist_dot(ac, ap);
        const float d3 = dist_dot(ab, bp), d4 = dist_dot(ac, bp);
        const float d5 = dist_dot(ab, cp), d6 = dist_dot(ac, cp);
        const float vc = FS(FM(d1, d4), FM(d3, d2));
        const float vb = FS(FM(d5, d2), FM(d1, d6));
        const float va = FS(FM(d3, d6), FM(d5, d4));
        const float e43 = FS(d4, d3), e56 = FS(d5, d6);
        float num = 0.0f, den = 1.0f;
        if (d1 <= 0.0f && d2 <= 0.0f) region = 0;
        else if (d3 >= 0.0f && d4 <= d3) region = 1;
        else if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) { region = 3; num = d1; den = FS(d1, d3); }
        else if (d6 >= 0.0f && d5 <= d6) region = 2;
        else if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) { region = 4; num = d2; den = FS(d2, d6); }
        else if (va <= 0.0f && e43 >= 0.0f && e56 >= 0.0f) { region = 5; num = e43; den = FA(e43, e56); }
        else { region = 6; den = FA(FA(va, vb), vc); }
        if (!(den > 0.0f)) edges = true;
        else if (region == 6)
        {
            const float r = FD(1.0f, den);
            vi = FM(vb, r); wi = FM(vc, r);
            if (!(vi >= 0.0f && wi >= 0.0f && FA(vi, wi) <= 1.0f)) edges = true;
        }
        else if (region >= 3) s = FD(num, den);
    }
    float de = 0.0f;
    if (edges || sliver) de = fminf(fminf(dist_seg_d2(p, a, b), dist_seg_d2(p, b, c)), dist_seg_d2(p, c, a));
    if (edges) return de;
    float d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        float q;
        switch (region)
        {
        case 0: q = a[k]; break;
        case 1: q = b[k]; break;
        case 2: q = c[k]; break;
        case 3: q = FA(a[k], FM(s, ab[k])); break;
        case 4: q = FA(a[k], FM(s, ac[k])); break;
        case 5: q = FA(b[k], FM(s, bc[k])); break;
        default: q = FA(FA(a[k], FM(ab[k], vi)), FM(ac[k], wi)); break;
        }
        d[k] = FS(p[k], q);
    }
    const float dq = dist_dot(d, d);
    return sliver ? fminf(dq, de) : dq;
}

__device__ __forceinline__ int dist_cell(float x, float lo, float h, int n)
{
    float v = FD(FS(x, lo), h);
    v = fminf(fmaxf(v, 0.0f), static_cast<float>(n - 1));
    return static_cast<int>(floorf(v));
}

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

// The nearest face of m to p within lim2 = max_distance^2: (bd2, bf), or (+inf, -1); tests counts the point-triangle evaluations
__device__ __forceinline__ void dist_nearest(const float* p, const DistMesh& m, const DistGrid& g, float lim2, float& bd2, int& bf, long long& tests)
{
    int c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = dist_cell(p[k], g.lo[k], g.h, g.n[k]);
    const double margin = g.margin + ldexp(static_cast<double>(fmaxf(fmaxf(fabsf(p[0]), fabsf(p[1])), fabsf(p[2]))), -16);
    bd2 = __int_as_float(0x7f800000); bf = -1;
#pragma unroll 1
    for (int r = 0;; ++r)
    {
        const int z0 = max(c[2] - r, 0), z1 = min(c[2] + r, g.n[2] - 1), y0 = max(c[1] - r, 0), y1 = min(c[1] + r, g.n[1] - 1);
#pragma unroll 1
        for (int z = z0; z <= z1; ++z)
#pragma unroll 1
            for (int y = y0; y <= y1; ++y)
            {
                const bool full = r == 0 || z == c[2] - r || z == c[2] + r || y == c[1] - r || y == c[1] + r;
                const int step = full ? 1 : 2 * r;
#pragma unroll 1
                for (int x = c[0] - r; x <= c[0] + r; x += step)
                {
                    if (x < 0 || x >= g.n[0]) continue;
                    const int64_t cell = (static_cast<int64_t>(z) * g.n[1] + y) * g.n[0] + x;
                    const int64_t e0 = g.off[cell], e1 = e0 + g.cnt[cell];
#pragma unroll 1
                    for (int64_t e = e0; e < e1; ++e)
                    {
                        const int f = g.faces[e];
                        const int3 fv = m.faces[f];
                        ++tests;
                        const float d2 = dist_point_tri_d2(p, m.vpos + 3 * static_cast<size_t>(fv.x), m.vpos + 3 * static_cast<size_t>(fv.y),
                                                           m.vpos + 3 * static_cast<size_t>(fv.z));
                        if (d2 <= lim2 && (d2 < bd2 || (d2 == bd2 && f < bf))) { bd2 = d2; bf = f; }
                    }
                }
            }
        double lb = 1e300;
        bool more = false;
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            if (c[k] - r > 0) { more = true; lb = fmin(lb, static_cast<double>(p[k]) - (static_cast<double>(g.lo[k]) + static_cast<double>(c[k] - r) * g.h)); }
            if (c[k] + r < g.n[k] - 1) { more = true; lb = fmin(lb, (static_cast<double>(g.lo[k]) + static_cast<double>(c[k] + r + 1) * g.h) - static_cast<double>(p[k])); }
        }
        if (!more) break;
        lb -= margin;
        const double lim = static_cast<double>(bf >= 0 ? bd2 : lim2);
        if (lb > 0.0 && lb * lb > lim) break;
    }
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
