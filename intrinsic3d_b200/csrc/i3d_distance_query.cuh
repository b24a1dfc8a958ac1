/*
 * i3d_distance_query.cuh — the point-triangle closest point and the nearest-face query through a uniform search grid, as stated in
 * i3d_distance.cuh.  No kernels: the distance module (i3d_distance.cuh) and the mesh-to-grid conversion (i3d_grid_from_mesh.cuh) both
 * include it, so the arithmetic is written down once and neither module compiles the other's kernels.
 */
#pragma once
#include "i3d_distance.h"
#include "i3d_grid.cuh"

namespace i3d
{

// A triangle with dot(n, n) <= 2^-20 dot(ab, ab) dot(ac, ac) (an angle below about 1e-3 rad) is a sliver: the float signs of Ericson's
// region tests cancel there, so its d^2 is also bounded by its edges'
constexpr float kDistSliver = 9.5367431640625e-07f;

// The feature of a triangle (a, b, c) a closest point lies on
enum { DIST_VERTEX_A = 0, DIST_VERTEX_B, DIST_VERTEX_C, DIST_EDGE_AB, DIST_EDGE_AC, DIST_EDGE_BC, DIST_INTERIOR };

__device__ __forceinline__ float dist_dot(const float* x, const float* y) { return FA(FA(FM(x[0], y[0]), FM(x[1], y[1])), FM(x[2], y[2])); }

// d^2 from p to segment s0 s1; with dv set, also p - q into dv and the clamped parameter into *t
__device__ __forceinline__ float dist_seg_d2(const float* p, const float* s0, const float* s1, float* dv = nullptr, float* tq = nullptr)
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
    if (dv)
    {
#pragma unroll
        for (int k = 0; k < 3; ++k) dv[k] = d[k];
        *tq = t;
    }
    return dist_dot(d, d);
}

// The feature of the point at t on segment (v0, v1) of a triangle: its end vertex at t = 0 or 1, else the edge
__device__ __forceinline__ int dist_seg_feature(float t, int v0, int v1, int edge) { return t == 0.0f ? v0 : (t == 1.0f ? v1 : edge); }

// float d^2 from p to triangle (a, b, c) (the rule at the top of i3d_distance.cuh).  With feature set, also the feature the closest
// point lies on and p - q into dv: the procedure's region; for the edge fallback the segment of the minimum (ties to ab, then bc, then
// ca) and dist_seg_feature of its t; for a sliver the procedure's when its d^2 <= the edges', else the segment's.
__device__ __forceinline__ float dist_point_tri(const float* p, const float* a, const float* b, const float* c, int* feature, float* dv)
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
    int fe = 0;
    float dve[3] = {0.0f, 0.0f, 0.0f};
    if (edges || sliver)
    {
        if (feature)
        {
            float d0[3], d1[3], d2[3], t0, t1, t2;
            const float e0 = dist_seg_d2(p, a, b, d0, &t0), e1 = dist_seg_d2(p, b, c, d1, &t1), e2 = dist_seg_d2(p, c, a, d2, &t2);
            de = fminf(fminf(e0, e1), e2);
            const int w = (e0 <= e1 && e0 <= e2) ? 0 : (e1 <= e2 ? 1 : 2);
            const float* dw = w == 0 ? d0 : (w == 1 ? d1 : d2);
#pragma unroll
            for (int k = 0; k < 3; ++k) dve[k] = dw[k];
            fe = w == 0 ? dist_seg_feature(t0, DIST_VERTEX_A, DIST_VERTEX_B, DIST_EDGE_AB)
                        : (w == 1 ? dist_seg_feature(t1, DIST_VERTEX_B, DIST_VERTEX_C, DIST_EDGE_BC) : dist_seg_feature(t2, DIST_VERTEX_C, DIST_VERTEX_A, DIST_EDGE_AC));
        }
        else de = fminf(fminf(dist_seg_d2(p, a, b), dist_seg_d2(p, b, c)), dist_seg_d2(p, c, a));
    }
    if (edges)
    {
        if (feature)
        {
            *feature = fe;
#pragma unroll
            for (int k = 0; k < 3; ++k) dv[k] = dve[k];
        }
        return de;
    }
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
    if (feature)
    {
        const bool proc = !sliver || dq <= de;
        *feature = proc ? region : fe;
#pragma unroll
        for (int k = 0; k < 3; ++k) dv[k] = proc ? d[k] : dve[k];
    }
    return sliver ? fminf(dq, de) : dq;
}

// float d^2 from p to triangle (a, b, c)
__device__ __forceinline__ float dist_point_tri_d2(const float* p, const float* a, const float* b, const float* c)
{
    return dist_point_tri(p, a, b, c, nullptr, nullptr);
}

__device__ __forceinline__ int dist_cell(float x, float lo, float h, int n)
{
    float v = FD(FS(x, lo), h);
    v = fminf(fmaxf(v, 0.0f), static_cast<float>(n - 1));
    return static_cast<int>(floorf(v));
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

} // namespace i3d
