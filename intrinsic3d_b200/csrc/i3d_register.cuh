/*
 * i3d_register.cuh — registering the reference mesh B to the resident mesh A (DESIGN.md §6aa): point-to-plane ICP of A's area samples
 * against B's faces.  Restated in numpy by tests/register_ref.py.  FM / FA / FS / FD are one IEEE float operation each, the double
 * operations are explicit __d*_rn (no contraction).
 *
 * Unknown.  T maps B onto A: x_A = R x_B + t, 12 doubles R row-major | t (the tracker's pose layout).  The state is M = T^-1 (A's frame ->
 * B's frame) in a TrackState: k_track_init(T_init) sets it (it inverts its input), k_track_solve updates it (M <- [Rodrigues(w) | v] M),
 * and its w2c is then the T returned.  B and its search grid do not move during a call; the grid is planned once with the first (largest)
 * stage distance.
 *
 * Samples.  Every face of A at its L^2 sub-triangle centroids with weight double(area) / L^2 (dist_sample's rule and order, one thread
 * per sample); a zero-area face drops its samples.  p' = tr_xform(Mf, Mf + 9, P), Mf the float copy of M.
 *
 * Correspondence.  The nearest face of B to p' within the stage's max_distance (dist_nearest: the lexicographic minimum of (d^2, face)),
 * its p' - q as dist_point_tri returns it (dv), and c = FS(p', dv) per coordinate.  A face's unit normal u = n / __fsqrt_rn(dot(n, n)),
 * n = (v1 - v0) x (v2 - v0) in dist_sample's operations, and 0 when that length is 0; n_B = u of B's face, n_A = tr_xform(Mf, u of A's
 * face).  The row is kept when the sample is matched, n_A and n_B are both non-zero and, when min_normal_cos > -1, dist_dot(n_A, n_B) >=
 * min_normal_cos (a thin wall does not match its back side).
 *
 * Row.  In double from the float values: r = ((nB0 (p'0 - c0) + nB1 (p'1 - c1)) + nB2 (p'2 - c2)), J = [p' x n_B, n_B] (the tracker's
 * order); the 29 values are (w J_a) J_b (upper triangle, row by row), (w J_a) r, (w r) r and 1, so slot 28 counts rows as k_track_solve
 * expects.  Area weights make the system independent of how finely A is tessellated.
 *
 * Sums.  Per block dist_block_reduce<kTrackVals> (a warp shuffle tree, then the warps in order), then k_tile_sums<kTrackVals> adds the
 * blocks in order; sum w goes the same way per block (dist_block_reduce<1>) for the first and the last system and its blocks are added
 * in order on the host.  No float atomics: every result is bit-identical from run to run.
 *
 * Transform (k_reg_transform).  x <- __double2float_rn(((R0 x0 + R1 x1) + R2 x2) + t) per row of R, in double from the float x.
 */
#pragma once
#include "i3d_distance.cuh"
#include "i3d_track.h"

namespace i3d
{

struct RegQuery
{
    int L;
    float max_distance;         // of the stage
    float min_cos;
    int use_cos;
};

// The unit face normal of face f of m (0 for a zero-length normal)
__device__ __forceinline__ void reg_face_normal(const DistMesh& m, int64_t f, float u[3])
{
    const int3 fv = m.faces[f];
    const float* p0 = m.vpos + 3 * static_cast<size_t>(fv.x);
    const float* p1 = m.vpos + 3 * static_cast<size_t>(fv.y);
    const float* p2 = m.vpos + 3 * static_cast<size_t>(fv.z);
    float e1[3], e2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { e1[k] = FS(p1[k], p0[k]); e2[k] = FS(p2[k], p0[k]); }
    const float n[3] = {FS(FM(e1[1], e2[2]), FM(e1[2], e2[1])), FS(FM(e1[2], e2[0]), FM(e1[0], e2[2])), FS(FM(e1[0], e2[1]), FM(e1[1], e2[0]))};
    const float len = __fsqrt_rn(dist_dot(n, n));
#pragma unroll
    for (int k = 0; k < 3; ++k) u[k] = len > 0.0f ? FD(n[k], len) : 0.0f;
}

__device__ __forceinline__ bool reg_nonzero(const float* v) { return v[0] != 0.0f || v[1] != 0.0f || v[2] != 0.0f; }

// One thread per sample of a at the pose of *state: the system's block partials [blocks][kTrackVals], with wpartials the blocks' sum w
// [blocks], with keep_face the per-sample nearest face (-1: none or a zero-area face); the point-triangle tests are added to *tests_total.
// Bounded to two blocks per SM like k_dist_samples: three would leave 80 registers and spill.
__global__ void __launch_bounds__(kThreads, 2) k_reg_rows(DistMesh a, DistMesh b, DistGrid g, RegQuery q, const TrackState* __restrict__ state,
                                                       int32_t* __restrict__ keep_face, double* __restrict__ partials, double* __restrict__ wpartials,
                                                       unsigned long long* __restrict__ tests_total)
{
    const int LL = q.L * q.L;
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    float area = 0.0f, p[3] = {0.0f, 0.0f, 0.0f}, c[3] = {0.0f, 0.0f, 0.0f}, nb[3] = {0.0f, 0.0f, 0.0f};
    bool keep = false;
    long long tests = 0;
    if (t < a.F * LL)
    {
        const int64_t f = t / LL;
        float P[3];
        dist_sample(a, f, static_cast<int>(t - f * LL), q.L, P, area);
        int bf = -1;
        if (area > 0.0f)
        {
            float Mf[12];
#pragma unroll
            for (int i = 0; i < 12; ++i) Mf[i] = state->Tf[i];
            tr_xform(Mf, Mf + 9, P, p);
            float bd2;
            dist_nearest(p, b, g, FM(q.max_distance, q.max_distance), bd2, bf, tests);
            if (bf >= 0)
            {
                const int3 fv = b.faces[bf];
                float dv[3];
                int feature;
                dist_point_tri(p, b.vpos + 3 * static_cast<size_t>(fv.x), b.vpos + 3 * static_cast<size_t>(fv.y), b.vpos + 3 * static_cast<size_t>(fv.z),
                               &feature, dv);
#pragma unroll
                for (int k = 0; k < 3; ++k) c[k] = FS(p[k], dv[k]);
                float ua[3], na[3];
                reg_face_normal(b, bf, nb);
                reg_face_normal(a, f, ua);
                tr_xform(Mf, nullptr, ua, na);
                keep = reg_nonzero(na) && reg_nonzero(nb) && (!q.use_cos || dist_dot(na, nb) >= q.min_cos);
            }
        }
        if (keep_face) keep_face[t] = bf;
    }
    // the values are formed after the search, so that they are not live across it
    double v[kTrackVals], w = 0.0;
#pragma unroll
    for (int j = 0; j < kTrackVals; ++j) v[j] = 0.0;
    if (keep)
    {
        w = __ddiv_rn(static_cast<double>(area), static_cast<double>(LL));
        double pd[3], nd[3], J[6];
#pragma unroll
        for (int k = 0; k < 3; ++k) { pd[k] = static_cast<double>(p[k]); nd[k] = static_cast<double>(nb[k]); }
        const double r = __dadd_rn(__dadd_rn(__dmul_rn(nd[0], __dsub_rn(pd[0], static_cast<double>(c[0]))),
                                             __dmul_rn(nd[1], __dsub_rn(pd[1], static_cast<double>(c[1])))),
                                   __dmul_rn(nd[2], __dsub_rn(pd[2], static_cast<double>(c[2]))));
        J[0] = __dsub_rn(__dmul_rn(pd[1], nd[2]), __dmul_rn(pd[2], nd[1]));
        J[1] = __dsub_rn(__dmul_rn(pd[2], nd[0]), __dmul_rn(pd[0], nd[2]));
        J[2] = __dsub_rn(__dmul_rn(pd[0], nd[1]), __dmul_rn(pd[1], nd[0]));
        J[3] = nd[0]; J[4] = nd[1]; J[5] = nd[2];
        int j = 0;
#pragma unroll
        for (int x = 0; x < 6; ++x)
        {
            const double wj = __dmul_rn(w, J[x]);
#pragma unroll
            for (int y = x; y < 6; ++y, ++j) v[j] = __dmul_rn(wj, J[y]);
            v[21 + x] = __dmul_rn(wj, r);
        }
        v[27] = __dmul_rn(__dmul_rn(w, r), r);
        v[28] = 1.0;
    }
    dist_block_reduce<kTrackVals>(v, 0u, partials);
    if (wpartials) dist_block_reduce<1>(&w, 0u, wpartials);
    unsigned long long n = static_cast<unsigned long long>(tests);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(tests_total, n);
}

// One thread per vertex: x <- float(R x + t) in double (T [12] R row-major | t)
__global__ void k_reg_transform(int64_t V, float* __restrict__ vpos, const double* __restrict__ T)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= V) return;
    float* p = vpos + 3 * i;
    const double x[3] = {static_cast<double>(p[0]), static_cast<double>(p[1]), static_cast<double>(p[2])};
#pragma unroll
    for (int d = 0; d < 3; ++d)
        p[d] = __double2float_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[3 * d], x[0]), __dmul_rn(T[3 * d + 1], x[1])), __dmul_rn(T[3 * d + 2], x[2])), T[9 + d]));
}

} // namespace i3d
