/*
 * i3d_raster.cuh — the resident mesh rasterized into the keyframes and into new views (DESIGN.md §6w): per pixel the nearest face, its
 * depth, barycentrics, normal and colour, and per keyframe the depth and colour error against the frame.  Restated in numpy float32 by
 * tests/raster_ref.py.  FM / FA / FS / FD: one IEEE float operation each, no contraction.
 *
 * Per pixel:
 *   ray      pixel (u, v) -> (x, y) by pixel_ray (i3d_pixel_ray.cuh, the renderer's rule); the camera ray is d = (x, y, 1) from the origin.
 *   vertex   q[k] = ((R[k][0] p0 + R[k][1] p1) + R[k][2] p2) + t[k], the camera-space vertex from the float R | t.
 *   hit      a face with every camera z <= 0 is a miss; otherwise the watertight test of Woop, Benthin & Wald (2013): kz = the dominant axis of d (|x| > |y| ? (|x| > 1 ? x : z) : (|y| > 1 ?
 *            y : z)), kx = kz + 1, ky = kx + 1 (mod 3), swapped when d[kz] < 0; Sx = d[kx] / d[kz], Sy = d[ky] / d[kz], Sz = 1 / d[kz];
 *            per vertex P in (A, B, C) = (q0, q1, q2): Px = P[kx] - Sx P[kz], Py = P[ky] - Sy P[kz];
 *            U = Cx By - Cy Bx, V = Ax Cy - Ay Cx, W = Bx Ay - By Ax; when any of them is exactly 0 all three are recomputed in double from
 *            the float operands (exact products, one rounded difference) and rounded to float;
 *            a miss when (U < 0 or V < 0 or W < 0) and (U > 0 or V > 0 or W > 0), or det = (U + V) + W is 0;
 *            T = ((U Sz A[kz]) + (V Sz B[kz])) + (W Sz C[kz]) (each product as U (Sz A[kz])), t = T / det, a hit needs t > 0;
 *            a = V / det (weight of v1), b = W / det (weight of v2), w0 = (1 - a) - b.  Since d_z = 1, t is the camera z.
 *            No culling: either orientation hits.  NaN anywhere gives a miss.
 *   winner   the lexicographic minimum of (t, face id) over all faces: a 64-bit atomicMin of float_as_uint(t) << 32 | face (t > 0, so
 *            the bits order like the floats).  The result does not depend on binning or launch order.
 *   shade    the winner's hit recomputed by the same function.  depth = t; face; bary = (a, b); normal = n / |n|, n = (v1 - v0) x (v2 -
 *            v0) with each component (e1[p] e2[q]) - (e1[q] e2[p]), |n| = __fsqrt_rn((n0 n0 + n1 n1) + n2 n2), (0, 0, 0) when |n| = 0
 *            (the texture bake's normal).
 *   colour   vertex: per channel trunc(clamp(((w0 c0 + a c1) + b c2) + 1/2, 0, 255)) (the bake's fallback rule).
 *            texture: (a, b) clamped as tex_bary does (negatives to 0, both divided by s = a + b when s > 1), w = (1 - a) - b, the
 *            face's cell-local UV corners (tex_corner) blended as u = (w u0 + a u1) + b u2 (v alike), and interp_u8 of the atlas at
 *            ((col S + u) - 1/2, (row S + v) - 1/2), cell c = face / 2 at column c % cols, row c / cols.  The clamped point lies in the
 *            face's UV triangle, so by the atlas's no-bleed property (i3d_texture.cuh) the lookup reads only texels the face owns.
 *   relit    (DESIGN.md §6x) the texture source's (a, b) clamping and (X, Y); A = interp_f32 of the decomposition's albedo atlas at (X, Y)
 *            (the same taps and weights as interp_u8, so the no-bleed property holds); P = (w0 p0 + a p1) + b p2 at the clamped (a, b);
 *            s' = sh_dot(normal, SH(P)) under the lighting of i3d_set_relight (sh_light_at); per channel trunc(clamp(((A s') 255) + 1/2,
 *            0, 255)); 0 for a zero normal.
 *
 * Statistics (keyframes): per pixel covered = hit, observed = frame depth > 0; a depth pair (covered and observed) adds |e| and e^2,
 * e = double(t) - double(z_frame), summed in double by a fixed tree over the 16 x 16 block and then the blocks in order (k_rast_sums),
 * so a view's bytes do not depend on the batch; a colour pair (covered, with a colour source) adds |e| and e^2 per channel, e = rendered
 * - frame (R, G, B against the frame's channels 2, 1, 0) as exact integers (integer atomics).
 *
 * Binning (free: it only decides which (pixel, face) pairs are tested).  The ray table holds every pixel's (x, y); 8 x 8 tiles keep the
 * box of their rays; tile rows and columns keep monotone envelopes of their bands (suffix minimum of the low ends, prefix maximum of the
 * high ends), so the rows and columns a box can touch are one contiguous range found by bisection.  Per (face, view): faces with every
 * camera z <= 0 are dropped (rast_hit misses them by its first rule); faces with some z <= 0, or whose
 * projected box is not finite, go to every tile and test every pixel ("straddling"); the others test the pixels of the tiles their
 * padded box of (X / Z, Y / Z) meets whose ray lies in that box.
 * Padding.  In exact arithmetic a ray that meets the triangle lies in the box of the projected vertices.  The float test sees the
 * sheared vertices with an error of at most ~2 eps (|X / Z| + |x|) z each (eps = 2^-24) and decides each edge function's sign up to
 * a relative error of ~3 eps, i.e. up to ~4 eps (M + E) in normalised coordinates, M the largest |coordinate| of the box and E its
 * largest side.  The pad 2^-12 (1 + M + E) exceeds that by a factor above 10^3, so binning never drops a pixel the float test would
 * accept.  i3d_debug_set_raster_binning(e, 0) sends every face to every tile and tests every pixel; the bytes are the same.
 */
#pragma once
#include "i3d_observe.cuh"
#include "i3d_pixel_ray.cuh"
#include "i3d_raster.h"
#include "i3d_texture_layout.cuh"

namespace i3d
{

// The binning pass of one batch of views: view z of the batch is view v0 + z of the call
struct RastBin
{
    int v0, W, H, TX, TY;
    const int32_t* ids; const float* Rt;
    const float2* rays; const float4* tbox; const float2* rowband; const float2* colband;
    unsigned long long* keys;           // [batch][H][W], ~0 = no face
    int binning;
    unsigned long long* counters;       // [0] pairs, [1] straddling, [2] behind, [3] tests
};

// The shading pass of one batch
struct RastShade
{
    int v0, W, H;
    const int32_t* ids; const float* Rt;
    const unsigned long long* keys; const float2* rays;
    const float* depth; const uint8_t* bgr;       // keyframes: the frames (bgr nullptr: no colour pairs); views: nullptr
    int color_source;
    float* out_depth; int32_t* out_face; float* out_bary; float* out_normal; uint8_t* out_rgb;
    double* partials;                   // [batch][tiles16][kRastSums]
    unsigned long long* counts;         // [n][kRastCounts] of the call
};

// The relit colour source's inputs: the albedo atlas [tex_H][tex_W][3] of the texture's decomposition and the lighting of i3d_set_relight
struct RastRelit
{
    const float* albedo;
    ShLight light;
};

__device__ __forceinline__ float rast_sel(const float (&a)[3], int k) { return k == 0 ? a[0] : (k == 1 ? a[1] : a[2]); }

__device__ __forceinline__ const float* rast_pose(const int32_t* ids, const float* Rt, int view)
{
    return Rt + 12 * static_cast<size_t>(ids ? ids[view] : view);
}

// The camera-space vertices of face f
__device__ __forceinline__ void rast_vertices(const RastMesh& m, int f, const float* __restrict__ Rt, float (&q)[3][3])
{
    const int3 fv = m.faces[f];
    const int vi[3] = {fv.x, fv.y, fv.z};
#pragma unroll
    for (int j = 0; j < 3; ++j)
    {
        const float* p = m.vpos + 3 * static_cast<size_t>(vi[j]);
        const float p0 = p[0], p1 = p[1], p2 = p[2];
#pragma unroll
        for (int k = 0; k < 3; ++k) q[j][k] = FA(FA(FA(FM(Rt[3 * k], p0), FM(Rt[3 * k + 1], p1)), FM(Rt[3 * k + 2], p2)), Rt[9 + k]);
    }
}

// The watertight ray-triangle test of the ray (x, y, 1) against camera-space vertices q (header): true with t > 0 and (a, b) on a hit
__device__ __forceinline__ bool rast_hit(const float (&q)[3][3], float x, float y, float& t, float& a, float& b)
{
    if (q[0][2] <= 0.0f && q[1][2] <= 0.0f && q[2][2] <= 0.0f) return false;    // no point of the face lies in front of the camera
    const float ax = fabsf(x), ay = fabsf(y);
    const int kz = ax > ay ? (ax > 1.0f ? 0 : 2) : (ay > 1.0f ? 1 : 2);
    int kx = kz == 2 ? 0 : kz + 1;
    int ky = kx == 2 ? 0 : kx + 1;
    const float d[3] = {x, y, 1.0f};
    const float dz = rast_sel(d, kz);
    if (dz < 0.0f) { const int s = kx; kx = ky; ky = s; }
    const float Sx = FD(rast_sel(d, kx), dz), Sy = FD(rast_sel(d, ky), dz), Sz = FD(1.0f, dz);
    float px[3], py[3], pz[3];
#pragma unroll
    for (int j = 0; j < 3; ++j)
    {
        const float zk = rast_sel(q[j], kz);
        px[j] = FS(rast_sel(q[j], kx), FM(Sx, zk));
        py[j] = FS(rast_sel(q[j], ky), FM(Sy, zk));
        pz[j] = FM(Sz, zk);
    }
    float U = FS(FM(px[2], py[1]), FM(py[2], px[1]));
    float V = FS(FM(px[0], py[2]), FM(py[0], px[2]));
    float W = FS(FM(px[1], py[0]), FM(py[1], px[0]));
    if (U == 0.0f || V == 0.0f || W == 0.0f)
    {
        const double Ax = px[0], Ay = py[0], Bx = px[1], By = py[1], Cx = px[2], Cy = py[2];
        U = __double2float_rn(__dsub_rn(__dmul_rn(Cx, By), __dmul_rn(Cy, Bx)));
        V = __double2float_rn(__dsub_rn(__dmul_rn(Ax, Cy), __dmul_rn(Ay, Cx)));
        W = __double2float_rn(__dsub_rn(__dmul_rn(Bx, Ay), __dmul_rn(By, Ax)));
    }
    if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) return false;
    const float det = FA(FA(U, V), W);
    if (!(det != 0.0f)) return false;
    const float T = FA(FA(FM(U, pz[0]), FM(V, pz[1])), FM(W, pz[2]));
    t = FD(T, det);
    if (!(t > 0.0f)) return false;
    a = FD(V, det);
    b = FD(W, det);
    return true;
}

// The ray table: (x, y) of every pixel
__global__ void k_rast_rays(RenderCam cam, int W, int H, float2* __restrict__ rays)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= static_cast<int64_t>(W) * H) return;
    const int v = static_cast<int>(i / W), u = static_cast<int>(i - static_cast<int64_t>(v) * W);
    float x, y;
    pixel_ray(cam, u, v, x, y);
    rays[i] = make_float2(x, y);
}

// Per 8 x 8 tile the box of its rays (x_lo, y_lo, x_hi, y_hi); non-finite rays are left out
__global__ void k_rast_tiles(int W, int H, int TX, int TY, const float2* __restrict__ rays, float4* __restrict__ tbox)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= TX * TY) return;
    const int ty = t / TX, tx = t - ty * TX;
    const float inf = __int_as_float(0x7f800000);
    float4 b = make_float4(inf, inf, -inf, -inf);
    for (int v = ty * kRastTile; v < min(H, (ty + 1) * kRastTile); ++v)
        for (int u = tx * kRastTile; u < min(W, (tx + 1) * kRastTile); ++u)
        {
            const float2 r = rays[static_cast<int64_t>(v) * W + u];
            b.x = fminf(b.x, r.x); b.y = fminf(b.y, r.y); b.z = fmaxf(b.z, r.x); b.w = fmaxf(b.w, r.y);
        }
    tbox[t] = b;
}

// The raw bands: block b < TY (32 threads) reduces tile row b to (min y_lo, max y_hi) into rowband[b], block TY + c column c to (min
// x_lo, max x_hi) into colband[c].  fminf / fmaxf are exact, so the order of the reduction does not matter.
__global__ void __launch_bounds__(32) k_rast_band_raw(int TX, int TY, const float4* __restrict__ tbox, float2* __restrict__ rowband,
                                                      float2* __restrict__ colband)
{
    const float inf = __int_as_float(0x7f800000);
    const bool row = static_cast<int>(blockIdx.x) < TY;
    const int k = row ? blockIdx.x : blockIdx.x - TY;
    const int m = row ? TX : TY;
    float lo = inf, hi = -inf;
    for (int i = threadIdx.x; i < m; i += 32)
    {
        const float4 b = tbox[row ? k * TX + i : i * TX + k];
        lo = fminf(lo, row ? b.y : b.x); hi = fmaxf(hi, row ? b.w : b.z);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if (threadIdx.x == 0) (row ? rowband : colband)[k] = make_float2(lo, hi);
}

// The monotone band envelopes of the raw bands, in place: rowband [TY] = (suffix min of the low ends, prefix max of the high ends),
// colband [TX] alike.  One block; thread 0 does the rows, thread 1 the columns (at most 1024 entries each).
__global__ void k_rast_bands(int TX, int TY, float2* __restrict__ rowband, float2* __restrict__ colband)
{
    if (threadIdx.x > 1) return;
    float2* band = threadIdx.x == 0 ? rowband : colband;
    const int n = threadIdx.x == 0 ? TY : TX;
    float hi = -__int_as_float(0x7f800000);
    for (int i = 0; i < n; ++i) { hi = fmaxf(hi, band[i].y); band[i].y = hi; }
    float lo = __int_as_float(0x7f800000);
    for (int i = n - 1; i >= 0; --i) { lo = fminf(lo, band[i].x); band[i].x = lo; }
}

// The contiguous range [i0, i1] of bands (monotone envelopes, n of them) that may meet [lo, hi]: the first with high end >= lo, the
// last with low end <= hi
__device__ __forceinline__ void rast_band_range(const float2* __restrict__ band, int n, float lo, float hi, int& i0, int& i1)
{
    int a = 0, b = n;                                  // first index with band.y >= lo
    while (a < b) { const int mid = (a + b) >> 1; if (band[mid].y >= lo) b = mid; else a = mid + 1; }
    i0 = a;
    a = 0; b = n;                                      // first index with band.x > hi
    while (a < b) { const int mid = (a + b) >> 1; if (band[mid].x > hi) b = mid; else a = mid + 1; }
    i1 = a - 1;
}

// One thread per (face, view of the batch in blockIdx.y): bin the face to tiles, test their pixels, atomicMin the winners' keys
__global__ void __launch_bounds__(kThreads) k_rast_faces(RastMesh m, RastBin rb)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    const int z = blockIdx.y;
    unsigned long long pairs = 0, tests = 0;
    unsigned straddling = 0, behind = 0;
    if (f < m.F)
    {
        const float* Rt = rast_pose(rb.ids, rb.Rt, rb.v0 + z);
        float q[3][3];
        rast_vertices(m, f, Rt, q);
        const int nb = (q[0][2] <= 0.0f) + (q[1][2] <= 0.0f) + (q[2][2] <= 0.0f);
        if (nb == 3 && rb.binning) behind = 1;
        else
        {
            float xlo = 0.0f, xhi = 0.0f, ylo = 0.0f, yhi = 0.0f;
            bool boxed = nb == 0;
            if (boxed)
            {
                const float X0 = FD(q[0][0], q[0][2]), X1 = FD(q[1][0], q[1][2]), X2 = FD(q[2][0], q[2][2]);
                const float Y0 = FD(q[0][1], q[0][2]), Y1 = FD(q[1][1], q[1][2]), Y2 = FD(q[2][1], q[2][2]);
                xlo = fminf(X0, fminf(X1, X2)); xhi = fmaxf(X0, fmaxf(X1, X2));
                ylo = fminf(Y0, fminf(Y1, Y2)); yhi = fmaxf(Y0, fmaxf(Y1, Y2));
                const float M = fmaxf(fmaxf(fabsf(xlo), fabsf(xhi)), fmaxf(fabsf(ylo), fabsf(yhi)));
                const float E = fmaxf(xhi - xlo, yhi - ylo);
                const float pad = (1.0f + M + E) * 2.44140625e-4f;     // 2^-12 (1 + M + E), see the header
                xlo -= pad; xhi += pad; ylo -= pad; yhi += pad;
                boxed = isfinite(xlo) && isfinite(xhi) && isfinite(ylo) && isfinite(yhi);
            }
            boxed = boxed && rb.binning;
            if (!boxed && nb > 0 && nb < 3) straddling = 1;
            else if (!boxed && nb == 0 && rb.binning) straddling = 1;      // a box that is not finite
            int r0 = 0, r1 = rb.TY - 1, c0 = 0, c1 = rb.TX - 1;
            if (boxed)
            {
                rast_band_range(rb.rowband, rb.TY, ylo, yhi, r0, r1);
                rast_band_range(rb.colband, rb.TX, xlo, xhi, c0, c1);
            }
            unsigned long long* keys = rb.keys + static_cast<int64_t>(z) * rb.W * rb.H;
            const unsigned long long fkey = static_cast<unsigned long long>(static_cast<unsigned>(f));
#pragma unroll 1
            for (int ty = r0; ty <= r1; ++ty)
#pragma unroll 1
                for (int tx = c0; tx <= c1; ++tx)
                {
                    if (boxed)
                    {
                        const float4 b = rb.tbox[ty * rb.TX + tx];
                        if (b.x > xhi || b.z < xlo || b.y > yhi || b.w < ylo) continue;
                    }
                    ++pairs;
                    const int u0 = tx * kRastTile, v0 = ty * kRastTile;
                    const int u1 = min(rb.W, u0 + kRastTile), v1 = min(rb.H, v0 + kRastTile);
#pragma unroll 1
                    for (int v = v0; v < v1; ++v)
#pragma unroll 1
                        for (int u = u0; u < u1; ++u)
                        {
                            const int64_t pix = static_cast<int64_t>(v) * rb.W + u;
                            const float2 r = rb.rays[pix];
                            if (boxed && !(r.x >= xlo && r.x <= xhi && r.y >= ylo && r.y <= yhi)) continue;
                            ++tests;
                            float t, a, b;
                            if (rast_hit(q, r.x, r.y, t, a, b))
                                atomicMin(keys + pix, (static_cast<unsigned long long>(__float_as_uint(t)) << 32) | fkey);
                        }
                }
        }
    }
    // integer warp sums, one atomic per warp and counter
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
    {
        pairs += __shfl_down_sync(0xffffffffu, pairs, o); tests += __shfl_down_sync(0xffffffffu, tests, o);
        straddling += __shfl_down_sync(0xffffffffu, straddling, o); behind += __shfl_down_sync(0xffffffffu, behind, o);
    }
    if ((threadIdx.x & 31) == 0)
    {
        if (pairs) atomicAdd(rb.counters, pairs);
        if (straddling) atomicAdd(rb.counters + 1, static_cast<unsigned long long>(straddling));
        if (behind) atomicAdd(rb.counters + 2, static_cast<unsigned long long>(behind));
        if (tests) atomicAdd(rb.counters + 3, tests);
    }
}

// The texture lookup of a hit of face f at (a, b): (a, b) clamped as tex_bary does into (ac, bc), the face's cell-local UV corners blended
// at w = (1 - ac) - bc, and the atlas position (X, Y) of the bilinear lookup (header)
__device__ __forceinline__ void rast_tex_lookup(const RastMesh& m, int f, float a, float b, float& ac, float& bc, float& X, float& Y)
{
    ac = a < 0.0f ? 0.0f : a; bc = b < 0.0f ? 0.0f : b;
    const float s = FA(ac, bc);
    if (s > 1.0f) { ac = FD(ac, s); bc = FD(bc, s); }
    const float w = FS(FS(1.0f, ac), bc);
    const bool fb = f & 1;
    float u0, v0, u1, v1, u2, v2;
    tex_corner(m.tex_S, fb, 0, u0, v0); tex_corner(m.tex_S, fb, 1, u1, v1); tex_corner(m.tex_S, fb, 2, u2, v2);
    const float u = FA(FA(FM(w, u0), FM(ac, u1)), FM(bc, u2));
    const float v = FA(FA(FM(w, v0), FM(ac, v1)), FM(bc, v2));
    const int cell = f >> 1;
    X = FS(FA(static_cast<float>((cell % m.tex_cols) * m.tex_S), u), 0.5f);
    Y = FS(FA(static_cast<float>((cell / m.tex_cols) * m.tex_S), v), 0.5f);
}

// The colour of a hit of face f at (a, b) from the colour source (header), R, G, B
__device__ __forceinline__ void rast_color(const RastMesh& m, int source, int f, float a, float b, uint8_t (&c)[3])
{
    if (source == I3D_RASTER_COLOR_VERTEX)
    {
        const int3 fv = m.faces[f];
        const float w0 = FS(FS(1.0f, a), b);
        const uint8_t* q0 = m.vcol + 3 * static_cast<size_t>(fv.x);
        const uint8_t* q1 = m.vcol + 3 * static_cast<size_t>(fv.y);
        const uint8_t* q2 = m.vcol + 3 * static_cast<size_t>(fv.z);
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            float x = FA(FA(FA(FM(w0, static_cast<float>(q0[k])), FM(a, static_cast<float>(q1[k]))), FM(b, static_cast<float>(q2[k]))), 0.5f);
            x = x < 0.0f ? 0.0f : (x > 255.0f ? 255.0f : x);
            c[k] = static_cast<uint8_t>(__float2int_rz(x));
        }
        return;
    }
    // texture (the statements of rast_tex_lookup, kept inline: calling it renumbers this instance's registers)
    float ac = a < 0.0f ? 0.0f : a, bc = b < 0.0f ? 0.0f : b;
    const float s = FA(ac, bc);
    if (s > 1.0f) { ac = FD(ac, s); bc = FD(bc, s); }
    const float w = FS(FS(1.0f, ac), bc);
    const bool fb = f & 1;
    float u0, v0, u1, v1, u2, v2;
    tex_corner(m.tex_S, fb, 0, u0, v0); tex_corner(m.tex_S, fb, 1, u1, v1); tex_corner(m.tex_S, fb, 2, u2, v2);
    const float u = FA(FA(FM(w, u0), FM(ac, u1)), FM(bc, u2));
    const float v = FA(FA(FM(w, v0), FM(ac, v1)), FM(bc, v2));
    const int cell = f >> 1;
    const float X = FS(FA(static_cast<float>((cell % m.tex_cols) * m.tex_S), u), 0.5f);
    const float Y = FS(FA(static_cast<float>((cell / m.tex_cols) * m.tex_S), v), 0.5f);
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = interp_u8(m.tex_rgb, m.tex_W, m.tex_H, X, Y, k);
}

// interp_u8's bilinear lookup on a float [h][w][3] image, without the truncation: taps (x0, y0), (x0, y1), (x1, y0), (x1, y1) with
// x0 = floor(x), x1 = x0 + 1 (y alike), weights w00 = (1 - fx)(1 - fy), w01 = (1 - fx) fy, w10 = fx (1 - fy), w11 = fx fy, fx = x - x0,
// out-of-image taps at weight 0; sum of w v over the taps with w > 0 in that order, over ((w00 + w10) + w01) + w11; 0 when that is 0
__device__ __forceinline__ float interp_f32(const float* __restrict__ img, int w, int h, float x, float y, int channel)
{
    const float fx0 = floorf(x), fy0 = floorf(y);
    const int x0 = static_cast<int>(fx0), y0 = static_cast<int>(fy0);
    const int x1 = x0 + 1, y1 = y0 + 1;
    float x1w = FS(x, fx0), y1w = FS(y, fy0);
    float x0w = FS(1.0f, x1w), y0w = FS(1.0f, y1w);
    if (x0 < 0 || x0 >= w) x0w = 0.0f;
    if (x1 < 0 || x1 >= w) x1w = 0.0f;
    if (y0 < 0 || y0 >= h) y0w = 0.0f;
    if (y1 < 0 || y1 >= h) y1w = 0.0f;
    const float w00 = FM(x0w, y0w), w10 = FM(x1w, y0w), w01 = FM(x0w, y1w), w11 = FM(x1w, y1w);
    const float sum_w = FA(FA(FA(w00, w10), w01), w11);
    float sum = 0.0f;
    if (w00 > 0.0f) sum = FA(sum, FM(img[(static_cast<size_t>(y0) * w + x0) * 3 + channel], w00));
    if (w01 > 0.0f) sum = FA(sum, FM(img[(static_cast<size_t>(y1) * w + x0) * 3 + channel], w01));
    if (w10 > 0.0f) sum = FA(sum, FM(img[(static_cast<size_t>(y0) * w + x1) * 3 + channel], w10));
    if (w11 > 0.0f) sum = FA(sum, FM(img[(static_cast<size_t>(y1) * w + x1) * 3 + channel], w11));
    if (!(sum_w > 0.0f)) return 0.0f;
    return FD(sum, sum_w);
}

// The relit colour of a hit of face f at (a, b) with unit face normal nrm (header): the albedo A at the texture source's lookup
// position, s' = sh_dot(nrm, SH(P)) at P = (w0 p0 + a p1) + b p2 of the clamped (a, b), per channel trunc(clamp((A s') 255 + 1/2, 0, 255));
// 0 for a zero normal
__device__ __forceinline__ void rast_relit(const RastMesh& m, const RastRelit& rl, int f, float a, float b, const float (&nrm)[3], uint8_t (&c)[3])
{
    if (nrm[0] == 0.0f && nrm[1] == 0.0f && nrm[2] == 0.0f) { c[0] = 0; c[1] = 0; c[2] = 0; return; }
    float ac, bc, X, Y;
    rast_tex_lookup(m, f, a, b, ac, bc, X, Y);
    const int3 fv = m.faces[f];
    const float* p0 = m.vpos + 3 * static_cast<size_t>(fv.x);
    const float* p1 = m.vpos + 3 * static_cast<size_t>(fv.y);
    const float* p2 = m.vpos + 3 * static_cast<size_t>(fv.z);
    const float w0 = FS(FS(1.0f, ac), bc);
    float P[3], sh[9];
#pragma unroll
    for (int k = 0; k < 3; ++k) P[k] = FA(FA(FM(w0, p0[k]), FM(ac, p1[k])), FM(bc, p2[k]));
    sh_light_at(rl.light, P, sh);
    const float s = sh_dot(nrm, sh);
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        float x = FA(FM(FM(interp_f32(rl.albedo, m.tex_W, m.tex_H, X, Y, k), s), 255.0f), 0.5f);
        x = x < 0.0f ? 0.0f : (x > 255.0f ? 255.0f : x);
        c[k] = static_cast<uint8_t>(__float2int_rz(x));
    }
}

// One thread per pixel, 16 x 16 blocks, views of the batch in gridDim.z: the planes and the statistics of the winners.  RELIT: the
// relit colour source (rast_relit) with its inputs as one more parameter (Relit = RastRelit), in an instance of its own so that the
// other sources' instance keeps its parameters and code.
template <bool RELIT, class... Relit>
__global__ void __launch_bounds__(kRenderTile * kRenderTile) k_rast_shade(RastMesh m, RastShade rs, Relit... relit)
{
    __shared__ double red[kRastSums][kRenderTile * kRenderTile];
    __shared__ unsigned s_cnt[kRenderTile * kRenderTile / 32][kRastCounts];
    const int u = blockIdx.x * kRenderTile + threadIdx.x, v = blockIdx.y * kRenderTile + threadIdx.y, z = blockIdx.z;
    const int view = rs.v0 + z;
    const int tid = threadIdx.y * kRenderTile + threadIdx.x;
    double sd[kRastSums] = {0.0, 0.0};
    unsigned cnt[kRastCounts];
#pragma unroll
    for (int j = 0; j < kRastCounts; ++j) cnt[j] = 0u;
    if (u < rs.W && v < rs.H)
    {
        const int64_t pix = static_cast<int64_t>(v) * rs.W + u;
        const unsigned long long key = rs.keys[static_cast<int64_t>(z) * rs.W * rs.H + pix];
        float t = 0.0f, a = 0.0f, b = 0.0f, nrm[3] = {0.0f, 0.0f, 0.0f};
        uint8_t c[3] = {0, 0, 0};
        int face = -1;
        bool hit = false;
        if (key != ~0ull)
        {
            face = static_cast<int>(key & 0xffffffffull);
            float q[3][3];
            rast_vertices(m, face, rast_pose(rs.ids, rs.Rt, view), q);
            const float2 r = rs.rays[pix];
            hit = rast_hit(q, r.x, r.y, t, a, b);          // the winner's own test: always a hit, with the key's t
            if (hit)
            {
                const int3 fv = m.faces[face];
                const float* p0 = m.vpos + 3 * static_cast<size_t>(fv.x);
                const float* p1 = m.vpos + 3 * static_cast<size_t>(fv.y);
                const float* p2 = m.vpos + 3 * static_cast<size_t>(fv.z);
                float e1[3], e2[3];
#pragma unroll
                for (int k = 0; k < 3; ++k) { e1[k] = FS(p1[k], p0[k]); e2[k] = FS(p2[k], p0[k]); }
                const float n0 = FS(FM(e1[1], e2[2]), FM(e1[2], e2[1]));
                const float n1 = FS(FM(e1[2], e2[0]), FM(e1[0], e2[2]));
                const float n2 = FS(FM(e1[0], e2[1]), FM(e1[1], e2[0]));
                const float len = __fsqrt_rn(FA(FA(FM(n0, n0), FM(n1, n1)), FM(n2, n2)));
                if (len > 0.0f) { nrm[0] = FD(n0, len); nrm[1] = FD(n1, len); nrm[2] = FD(n2, len); }
                if constexpr (RELIT) rast_relit(m, relit..., face, a, b, nrm, c);
                else if (rs.color_source != I3D_RASTER_COLOR_NONE) rast_color(m, rs.color_source, face, a, b, c);
            }
            else { face = -1; t = 0.0f; a = 0.0f; b = 0.0f; }
        }
        const int64_t op = static_cast<int64_t>(view) * rs.W * rs.H + pix;
        if (rs.out_depth) rs.out_depth[op] = t;
        if (rs.out_face) rs.out_face[op] = face;
        if (rs.out_bary) { rs.out_bary[2 * op] = a; rs.out_bary[2 * op + 1] = b; }
        if (rs.out_normal) { rs.out_normal[3 * op] = nrm[0]; rs.out_normal[3 * op + 1] = nrm[1]; rs.out_normal[3 * op + 2] = nrm[2]; }
        if (rs.out_rgb) { rs.out_rgb[3 * op] = c[0]; rs.out_rgb[3 * op + 1] = c[1]; rs.out_rgb[3 * op + 2] = c[2]; }
        cnt[0] = hit ? 1u : 0u;
        if (rs.depth)
        {
            const int f = rs.ids[view];
            const int64_t fp = static_cast<int64_t>(f) * rs.W * rs.H + pix;
            const float zo = rs.depth[fp];
            const bool obs = zo > 0.0f;
            cnt[1] = obs ? 1u : 0u;
            if (hit && obs)
            {
                const double dz = __dsub_rn(static_cast<double>(t), static_cast<double>(zo));
                cnt[2] = 1u; sd[0] = fabs(dz); sd[1] = __dmul_rn(dz, dz);
            }
            if (hit && rs.bgr && rs.color_source != I3D_RASTER_COLOR_NONE)
            {
                cnt[3] = 1u;
#pragma unroll
                for (int k = 0; k < 3; ++k)
                {
                    const int e = static_cast<int>(c[k]) - static_cast<int>(rs.bgr[3 * fp + 2 - k]);
                    cnt[4 + k] = static_cast<unsigned>(e < 0 ? -e : e);
                    cnt[7 + k] = static_cast<unsigned>(e * e);
                }
            }
        }
    }
    // per-block partials of the depth sums: a fixed tree over the block (as k_render_march)
#pragma unroll
    for (int j = 0; j < kRastSums; ++j) red[j][tid] = sd[j];
    // integer counts: warp sums (at most 32 * 255^2 each), then the block's warps, one atomic per block and count
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int j = 0; j < kRastCounts; ++j)
    {
        const unsigned w = __reduce_add_sync(0xffffffffu, cnt[j]);
        if (lane == 0) s_cnt[warp][j] = w;
    }
    __syncthreads();
    for (int w = kRenderTile * kRenderTile / 2; w > 0; w >>= 1)
    {
        if (tid < w)
        {
#pragma unroll
            for (int j = 0; j < kRastSums; ++j) red[j][tid] = __dadd_rn(red[j][tid], red[j][tid + w]);
        }
        __syncthreads();
    }
    const int tiles_x = gridDim.x, tiles_y = gridDim.y;
    const int64_t tile = (static_cast<int64_t>(z) * tiles_y + blockIdx.y) * tiles_x + blockIdx.x;
    if (tid < kRastSums) rs.partials[tile * kRastSums + tid] = red[tid][0];
    if (tid < kRastCounts)
    {
        unsigned long long s = 0;
        for (int w = 0; w < kRenderTile * kRenderTile / 32; ++w) s += s_cnt[w][tid];
        if (s) atomicAdd(rs.counts + static_cast<int64_t>(view) * kRastCounts + tid, s);
    }
}

// One thread per (view, value) of the batch: the view's blocks summed in order
__global__ void k_rast_sums(int n, int tiles, const double* __restrict__ partials, double* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * kRastSums) return;
    const int view = i / kRastSums, j = i % kRastSums;
    const double* p = partials + static_cast<int64_t>(view) * tiles * kRastSums + j;
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s = __dadd_rn(s, p[static_cast<int64_t>(t) * kRastSums]);
    out[i] = s;
}

} // namespace i3d
