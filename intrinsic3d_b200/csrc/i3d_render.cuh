/*
 * i3d_render.cuh — the surface rendered into the keyframes on the device (DESIGN.md §6m): one ray per pixel, marched through the device
 * voxel hash on a fixed lattice, with depth, normal, albedo, shading and intensity at the first sign change and the per-view depth and
 * photometric errors against the keyframe.
 *
 *   k_render_bounds   the bounding box of the voxel coordinates (integer atomics)
 *   k_render_bricks   the occupancy bitmap of 8^3 bricks over that box (integer atomics)
 *   k_render_march    one thread per pixel, 16 x 16 tiles, views in gridDim.z: planes + per-tile statistic partials
 *   k_live_bounds / k_live_bricks / k_render_march_live   the same three over the fusion volume in progress (DESIGN.md §6o): the voxels
 *                     with weight > 0, and the cube rule by one fusion-hash probe per corner (the volume has no neighbour table)
 *   k_render_march_color / k_render_march_live_color   the two marches with the model intensity plane of the tracker's photometric term
 *                     (DESIGN.md §6p): the voxel colours' intensities blended at the hit
 *   k_tile_sums       the fixed-order sum of a view's partials (also the tracker's)
 *
 * Compiled with the tracker in i3d_render.cu, which launches them (render::keyframes, i3d_render.h).  Every float
 * operation is explicitly rounded (no FMA contraction, IEEE division and square root), so the planes are byte-equal to tests/render_ref.py.
 * The statistics are double sums in a fixed order (tile tree, then tiles in order): a view's bytes depend only on that view.
 */
#pragma once
#include <limits.h>

#include "i3d_grid.cuh"
#include "i3d_pixel_ray.cuh"
#include "i3d_render.h"
#include "i3d_vis.cuh"

namespace i3d
{

__device__ __forceinline__ float rd_lerp(float a, float b, float t) { return FA(a, FM(t, FS(b, a))); }

// The cube of a point: base voxel (floor of p / voxel_size), the fractions in it and its 8 corners, corner i = dx + 2 dy + 4 dz.
struct RdCube { int32_t c[8]; float f[3]; int base[3]; };

enum { RD_INVALID = 0, RD_VALID = 1, RD_EMPTY_BRICK = 2 };

// The cube rule of k_mesh_classify: valid when all 8 corners exist with weight != 0; the neighbour table gives 7 corners, one hash probe
// the (1,1,1) corner.  With a bitmap, a base voxel in an empty brick is invalid without a probe (RD_EMPTY_BRICK: the march may skip).
__device__ __forceinline__ int rd_cube(const RenderGrid& rg, const float p[3], RdCube& q)
{
    const float vs = rg.g.voxel_size;
#pragma unroll
    for (int d = 0; d < 3; ++d)
    {
        const float gd = FD(p[d], vs);
        const float fl = floorf(gd);
        q.base[d] = __float2int_rz(fl);
        q.f[d] = FS(gd, fl);
    }
    if (rg.bricks)
    {
        int b[3];
#pragma unroll
        for (int d = 0; d < 3; ++d)
        {
            b[d] = q.base[d] - rg.blo[d];
            if (b[d] < 0) return RD_INVALID;
            b[d] >>= 3;
            if (b[d] >= rg.bdim[d]) return RD_INVALID;
        }
        const int64_t idx = (static_cast<int64_t>(b[2]) * rg.bdim[1] + b[1]) * rg.bdim[0] + b[0];
        if (!((rg.bricks[idx >> 5] >> (idx & 31)) & 1u)) return RD_EMPTY_BRICK;
    }
    const GridView& g = rg.g;
    const int32_t v = hash_find(rg.keys, rg.vals, rg.mask, q.base[0], q.base[1], q.base[2]);
    if (v < 0) return RD_INVALID;
    q.c[0] = v; q.c[1] = g.nbr[NB_XP * g.n + v]; q.c[2] = g.nbr[NB_YP * g.n + v]; q.c[3] = g.nbr[NB_XY * g.n + v];
    q.c[4] = g.nbr[NB_ZP * g.n + v]; q.c[5] = g.nbr[NB_XZ * g.n + v]; q.c[6] = g.nbr[NB_YZ * g.n + v];
#pragma unroll
    for (int i = 0; i < 7; ++i)
        if (q.c[i] < 0 || g.weight[q.c[i]] == 0.0f) return RD_INVALID;
    q.c[7] = hash_find(rg.keys, rg.vals, rg.mask, q.base[0] + 1, q.base[1] + 1, q.base[2] + 1);
    return (q.c[7] >= 0 && g.weight[q.c[7]] != 0.0f) ? RD_VALID : RD_INVALID;
}

// The same rule on the fusion volume in progress, which has no neighbour table: one probe of its hash per corner.  The base and brick
// steps are rd_cube's above, written out again because one shared helper for them adds 16 instructions to each of the four marches and
// slows k_render_march: i3d_render_keyframes (C3, statistics of all 200 keyframes, skipping on) took 106.3-106.9 ms as written here and
// 107.9-108.4 ms shared, and the C3 track_predict 112.6-113.1 ms against 114.4-114.9 ms (three alternating runs each, H100 80GB HBM3, 700 W).
__device__ __forceinline__ int rd_cube(const LiveGrid& lg, const float p[3], RdCube& q)
{
    const float vs = lg.voxel_size;
#pragma unroll
    for (int d = 0; d < 3; ++d)
    {
        const float gd = FD(p[d], vs);
        const float fl = floorf(gd);
        q.base[d] = __float2int_rz(fl);
        q.f[d] = FS(gd, fl);
    }
    if (lg.bricks)
    {
        int b[3];
#pragma unroll
        for (int d = 0; d < 3; ++d)
        {
            b[d] = q.base[d] - lg.blo[d];
            if (b[d] < 0) return RD_INVALID;
            b[d] >>= 3;
            if (b[d] >= lg.bdim[d]) return RD_INVALID;
        }
        const int64_t idx = (static_cast<int64_t>(b[2]) * lg.bdim[1] + b[1]) * lg.bdim[0] + b[0];
        if (!((lg.bricks[idx >> 5] >> (idx & 31)) & 1u)) return RD_EMPTY_BRICK;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
    {
        const int32_t c = fuse_find(lg.v.keys, lg.v.vals, lg.v.mask, q.base[0] + (i & 1), q.base[1] + ((i >> 1) & 1), q.base[2] + ((i >> 2) & 1));
        if (c < 0 || lg.v.weight[c] == 0.0f) return RD_INVALID;
        q.c[i] = c;
    }
    return RD_VALID;
}

__device__ __forceinline__ float rd_float(double a) { return __double2float_rn(a); }
__device__ __forceinline__ float rd_float(float a) { return a; }
// A voxel colour (R, G, B) as the frame store's level-0 intensity rule reads a pixel (k_frames_lum0): c = float(u8) * float(1/255) per
// channel, then (B 0.114 + G 0.587) + R 0.299 (DESIGN.md §6p)
__device__ __forceinline__ float rd_float(uchar4 c)
{
    const float inv = static_cast<float>(1.0 / 255.0);
    const float b = FM(static_cast<float>(c.z), inv), g = FM(static_cast<float>(c.y), inv), r = FM(static_cast<float>(c.x), inv);
    return FA(FA(FM(b, 0.114f), FM(g, 0.587f)), FM(r, 0.299f));
}

// Trilinear blend of float(a[c]) over the cube: along x, then y, then z.  s_out (optional) gets the 8 corner values.
template <class T>
__device__ __forceinline__ float rd_trilinear(const T* __restrict__ a, const RdCube& q, float (*s_out)[8] = nullptr)
{
    float s[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] = rd_float(a[q.c[i]]);
    if (s_out)
    {
#pragma unroll
        for (int i = 0; i < 8; ++i) (*s_out)[i] = s[i];
    }
    const float a00 = rd_lerp(s[0], s[1], q.f[0]), a10 = rd_lerp(s[2], s[3], q.f[0]);
    const float a01 = rd_lerp(s[4], s[5], q.f[0]), a11 = rd_lerp(s[6], s[7], q.f[0]);
    return rd_lerp(rd_lerp(a00, a10, q.f[1]), rd_lerp(a01, a11, q.f[1]), q.f[2]);
}

// The analytic gradient of the trilinear blend of the corner values s (grid units), normalised; (0,0,0) when its length is 0.
__device__ __forceinline__ void rd_normal(const float (&s)[8], const float f[3], float n[3])
{
    const float a00 = rd_lerp(s[0], s[1], f[0]), a10 = rd_lerp(s[2], s[3], f[0]);
    const float a01 = rd_lerp(s[4], s[5], f[0]), a11 = rd_lerp(s[6], s[7], f[0]);
    const float b0 = rd_lerp(a00, a10, f[1]), b1 = rd_lerp(a01, a11, f[1]);
    const float gx = rd_lerp(rd_lerp(FS(s[1], s[0]), FS(s[3], s[2]), f[1]), rd_lerp(FS(s[5], s[4]), FS(s[7], s[6]), f[1]), f[2]);
    const float gy = rd_lerp(FS(a10, a00), FS(a11, a01), f[2]);
    const float gz = FS(b1, b0);
    const float len = __fsqrt_rn(FA(FA(FM(gx, gx), FM(gy, gy)), FM(gz, gz)));
    if (len == 0.0f) { n[0] = n[1] = n[2] = 0.0f; return; }
    n[0] = FD(gx, len); n[1] = FD(gy, len); n[2] = FD(gz, len);
}

// The corners' per-voxel SH blended with the trilinear weights (wx * wy) * wz, renormalised over the corners that have SH.  False when
// no weight is left.
__device__ __forceinline__ bool rd_sh(const RenderGrid& rg, const RdCube& q, float sh[9])
{
    float wsum = 0.0f;
#pragma unroll
    for (int k = 0; k < 9; ++k) sh[k] = 0.0f;
#pragma unroll
    for (int i = 0; i < 8; ++i)
    {
        const int32_t c = q.c[i];
        if (!rg.sh_has[c]) continue;
        const float wx = (i & 1) ? q.f[0] : FS(1.0f, q.f[0]);
        const float wy = (i & 2) ? q.f[1] : FS(1.0f, q.f[1]);
        const float wz = (i & 4) ? q.f[2] : FS(1.0f, q.f[2]);
        const float w = FM(FM(wx, wy), wz);
#pragma unroll
        for (int k = 0; k < 9; ++k) sh[k] = FA(sh[k], FM(w, __double2float_rn(rg.g.sh[static_cast<int64_t>(k) * rg.g.n + c])));
        wsum = FA(wsum, w);
    }
    if (!(wsum > 0.0f)) return false;
#pragma unroll
    for (int k = 0; k < 9; ++k) sh[k] = FD(sh[k], wsum);
    return true;
}

// What the march reads besides the cube rule: the voxel size, the surface's sdf, the albedo at a hit and the per-voxel SH.  The volume in
// progress has only a float sdf.
__device__ __forceinline__ float rd_voxel_size(const RenderGrid& rg) { return rg.g.voxel_size; }
__device__ __forceinline__ float rd_voxel_size(const LiveGrid& lg) { return lg.voxel_size; }
__device__ __forceinline__ const double* rd_sdf(const RenderGrid& rg) { return rg.g.sdf; }
__device__ __forceinline__ const float* rd_sdf(const LiveGrid& lg) { return lg.v.sdf; }
__device__ __forceinline__ float rd_albedo(const RenderGrid& rg, const RdCube& q) { return rd_trilinear(rg.g.albedo, q); }
__device__ __forceinline__ float rd_albedo(const LiveGrid&, const RdCube&) { return 0.0f; }
__device__ __forceinline__ bool rd_sh(const LiveGrid&, const RdCube&, float*) { return false; }

// A grid G with the model intensity plane of the tracker's photometric term (DESIGN.md §6p): the voxel colours rgb (GridView::rgb of the
// installed grid, the Voxel colour array of the volume in progress, held here so that LiveGrid and FuseView keep their layout) and the
// output plane out_mi [n][H][W]
template <class G>
struct Colored : G
{
    const uchar4* rgb;
    float* out_mi;
};

// The march's model intensity output: nothing for a plain grid; for Colored<G> the trilinear blend of the corners' intensities
// (rd_float of the voxel colours) at the hit, 0 without one
template <class G>
__device__ __forceinline__ void rd_model_intensity(const G&, const RdCube&, bool, int64_t) {}
template <class G>
__device__ __forceinline__ void rd_model_intensity(const Colored<G>& cg, const RdCube& q, bool hit, int64_t pix)
{
    cg.out_mi[pix] = hit ? rd_trilinear(cg.rgb, q) : 0.0f;
}

// The point at ray parameter s
__device__ __forceinline__ void rd_point(const float o[3], const float dn[3], float s, float p[3])
{
#pragma unroll
    for (int d = 0; d < 3; ++d) p[d] = FA(o[d], FM(s, dn[d]));
}

// One thread per pixel (u, v) of view blockIdx.z.  Ray: the pixel centre through the inverse of obs_probe's projection (i3d_observe.cuh), in
// world coordinates; samples s_k = s0 + k * voxel_size / 2 from where the ray enters the voxel box (clipped to s >= 0) to where it
// leaves it; the hit is the first pair of consecutive valid samples going from > 0 to <= 0 whose linearly interpolated crossing lies in a
// valid cube.  G: the installed grid (RenderGrid), the fusion volume in progress (LiveGrid), or either with the model intensity plane
// (Colored<G>, rd_model_intensity).
template <class G>
__device__ __forceinline__ void rd_march(G rg, RenderCam cam, RenderViews rv)
{
    __shared__ double red[kRenderStats][kRenderTile * kRenderTile];
    const int u = blockIdx.x * kRenderTile + threadIdx.x, v = blockIdx.y * kRenderTile + threadIdx.y, view = blockIdx.z;
    const int tid = threadIdx.y * kRenderTile + threadIdx.x;
    double st[kRenderStats];
#pragma unroll
    for (int j = 0; j < kRenderStats; ++j) st[j] = 0.0;
    unsigned nsamp = 0;
    if (u < rv.W && v < rv.H)
    {
        const int f = rv.ids[view];
        const float* Rt = rv.Rt + 12 * f;
        // pixel -> normalised camera coordinates (i3d_pixel_ray.cuh)
        float x, y;
        pixel_ray(cam, u, v, x, y);
        // world ray: o = -R^T t, direction R^T (x, y, 1) normalised; camera z = s / |R^T (x, y, 1)|
        float o[3], dn[3];
#pragma unroll
        for (int d = 0; d < 3; ++d)
        {
            o[d] = -FA(FA(FM(Rt[d], Rt[9]), FM(Rt[3 + d], Rt[10])), FM(Rt[6 + d], Rt[11]));
            dn[d] = FA(FA(FM(Rt[d], x), FM(Rt[3 + d], y)), Rt[6 + d]);
        }
        const float len = __fsqrt_rn(FA(FA(FM(dn[0], dn[0]), FM(dn[1], dn[1])), FM(dn[2], dn[2])));
#pragma unroll
        for (int d = 0; d < 3; ++d) dn[d] = FD(dn[d], len);
        // the lattice: entry and exit of the voxel box (slab test), entry clipped to s >= 0
        float s0 = 0.0f, s1 = __int_as_float(0x7f800000);
        bool any = true;
#pragma unroll
        for (int d = 0; d < 3; ++d)
        {
            if (dn[d] != 0.0f)
            {
                const float ta = FD(FS(rg.lo[d], o[d]), dn[d]), tb = FD(FS(rg.hi[d], o[d]), dn[d]);
                s0 = fmaxf(s0, fminf(ta, tb));
                s1 = fminf(s1, fmaxf(ta, tb));
            }
            else if (o[d] < rg.lo[d] || o[d] > rg.hi[d]) any = false;
        }
        // a non-finite ray (a NaN or infinite pose) has no samples: fminf / fmaxf would drop its NaN bounds and leave [0, inf)
        bool finite = isfinite(s1);
#pragma unroll
        for (int d = 0; d < 3; ++d) finite = finite && isfinite(o[d]) && isfinite(dn[d]);
        const float h = FM(rd_voxel_size(rg), 0.5f);
        const auto* sdf = rd_sdf(rg);
        RdCube q;
        float s_hit = 0.0f;
        bool hit = false;
        if (any && finite && s0 <= s1)
        {
            bool prev_ok = false;
            float prev = 0.0f;
            for (int k = 0; k <= kRenderMaxLattice;)
            {
                const float s = FA(s0, FM(__int2float_rn(k), h));
                if (!(s <= s1)) break;
                ++nsamp;
                float p[3];
                rd_point(o, dn, s, p);
                const int r = rd_cube(rg, p, q);
                if (r == RD_EMPTY_BRICK)
                {
                    // jump to one sample before the ray leaves this brick: every sample up to there has its base in the brick
                    float te = __int_as_float(0x7f800000);
#pragma unroll
                    for (int d = 0; d < 3; ++d)
                    {
                        if (dn[d] == 0.0f) continue;
                        const int b0 = rg.blo[d] + ((q.base[d] - rg.blo[d]) & ~7);
                        const float face = FM(__int2float_rn(dn[d] > 0.0f ? b0 + 8 : b0), rd_voxel_size(rg));
                        te = fminf(te, FD(FS(face, o[d]), dn[d]));
                    }
                    const float kf = floorf(FD(FS(te, s0), h));
                    const int kn = kf < static_cast<float>(kRenderMaxLattice) ? static_cast<int>(kf) - 1 : kRenderMaxLattice;
                    prev_ok = false;
                    k = kn > k + 1 ? kn : k + 1;
                    continue;
                }
                if (r == RD_VALID)
                {
                    const float val = rd_trilinear(sdf, q);
                    if (prev_ok && prev > 0.0f && val <= 0.0f)
                    {
                        const float tau = FD(prev, FS(prev, val));
                        const float sc = FA(FA(s0, FM(__int2float_rn(k - 1), h)), FM(tau, h));
                        float pc[3];
                        rd_point(o, dn, sc, pc);
                        RdCube qc;
                        if (rd_cube(rg, pc, qc) == RD_VALID) { q = qc; s_hit = sc; hit = true; break; }
                    }
                    prev_ok = true; prev = val;
                }
                else prev_ok = false;
                ++k;
            }
        }
        // outputs at the hit
        float depth = 0.0f, nrm[3] = {0.0f, 0.0f, 0.0f}, alb = 0.0f, shade = 0.0f, inten = 0.0f;
        bool shade_ok = false;
        if (hit)
        {
            depth = FD(s_hit, len);
            float s8[8];
            rd_trilinear(sdf, q, &s8);
            rd_normal(s8, q.f, nrm);
            alb = rd_albedo(rg, q);
            if (rv.photometric)
            {
                float sh[9];
                if (rd_sh(rg, q, sh) && !(nrm[0] == 0.0f && nrm[1] == 0.0f && nrm[2] == 0.0f))
                {
                    shade_ok = true;
                    shade = vis_shading(nrm, sh, 1.0f);
                    inten = vis_shading(nrm, sh, alb);
                }
            }
        }
        const int64_t pix = (static_cast<int64_t>(view) * rv.H + v) * rv.W + u;
        if (rv.out_depth) rv.out_depth[pix] = depth;
        if (rv.out_normal) { rv.out_normal[3 * pix] = nrm[0]; rv.out_normal[3 * pix + 1] = nrm[1]; rv.out_normal[3 * pix + 2] = nrm[2]; }
        if (rv.out_albedo) rv.out_albedo[pix] = alb;
        if (rv.out_shading) rv.out_shading[pix] = shade;
        if (rv.out_intensity) rv.out_intensity[pix] = inten;
        rd_model_intensity(rg, q, hit, pix);
        // statistics against the keyframe
        const int64_t fp = (static_cast<int64_t>(f) * rv.H + v) * rv.W + u;
        const float zo = rv.depth[fp];
        const bool obs = zo > 0.0f;
        st[0] = hit ? 1.0 : 0.0;
        st[1] = obs ? 1.0 : 0.0;
        if (hit && obs)
        {
            const double dz = __dsub_rn(static_cast<double>(depth), static_cast<double>(zo));
            st[2] = 1.0; st[4] = fabs(dz); st[5] = __dmul_rn(dz, dz);
        }
        if (shade_ok && obs)
        {
            const double di = __dsub_rn(static_cast<double>(inten), static_cast<double>(rv.lum[fp]));
            st[3] = 1.0; st[6] = fabs(di); st[7] = __dmul_rn(di, di);
        }
    }
    // per-tile partials: a fixed tree over the block
#pragma unroll
    for (int j = 0; j < kRenderStats; ++j) red[j][tid] = st[j];
    __syncthreads();
    for (int w = kRenderTile * kRenderTile / 2; w > 0; w >>= 1)
    {
        if (tid < w)
        {
#pragma unroll
            for (int j = 0; j < kRenderStats; ++j) red[j][tid] = __dadd_rn(red[j][tid], red[j][tid + w]);
        }
        __syncthreads();
    }
    const int64_t tile = (static_cast<int64_t>(view) * rv.tiles_y + blockIdx.y) * rv.tiles_x + blockIdx.x;
    if (tid < kRenderStats) rv.partials[tile * kRenderStats + tid] = red[tid][0];
    // samples evaluated: integer warp sums, one atomic per warp
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nsamp += __shfl_down_sync(0xffffffffu, nsamp, o);
    if ((tid & 31) == 0 && nsamp) atomicAdd(rv.samples, static_cast<unsigned long long>(nsamp));
}

__global__ void __launch_bounds__(kRenderTile * kRenderTile) k_render_march(RenderGrid rg, RenderCam cam, RenderViews rv) { rd_march(rg, cam, rv); }

// The march of the fusion volume in progress (geometry only: albedo 0, no shading), for the tracker's prediction
__global__ void __launch_bounds__(kRenderTile * kRenderTile) k_render_march_live(LiveGrid lg, RenderCam cam, RenderViews rv) { rd_march(lg, cam, rv); }

// The tracker's prediction with the model intensity plane (DESIGN.md §6p), from the installed grid and from the volume in progress
__global__ void __launch_bounds__(kRenderTile * kRenderTile) k_render_march_color(Colored<RenderGrid> cg, RenderCam cam, RenderViews rv)
{
    rd_march(cg, cam, rv);
}
__global__ void __launch_bounds__(kRenderTile * kRenderTile) k_render_march_live_color(Colored<LiveGrid> cg, RenderCam cam, RenderViews rv)
{
    rd_march(cg, cam, rv);
}

// One thread per (view, value) of V per-tile values: the view's tiles summed in order.  V = kRenderStats (k_render_march's statistics),
// kTrackVals (k_track_rows' systems).
template <int V>
__global__ void k_tile_sums(int n, int tiles, const double* __restrict__ partials, double* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * V) return;
    const int view = i / V, j = i % V;
    const double* p = partials + static_cast<int64_t>(view) * tiles * V + j;
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s = __dadd_rn(s, p[static_cast<int64_t>(t) * V]);
    out[i] = s;
}

// Min / max of the coordinates per warp (__reduce_*_sync), then per block in shared memory, then one integer atomic per block and value.
// w: only the voxels with weight > 0 count (nullptr: all).
__device__ __forceinline__ void rd_bounds(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z,
                                          const float* __restrict__ w, int* box)
{
    __shared__ int part[6][kThreads / 32];
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const bool in = v < n && (!w || w[v] > 0.0f);
    int c[6];
    c[0] = in ? x[v] : INT_MAX; c[1] = in ? y[v] : INT_MAX; c[2] = in ? z[v] : INT_MAX;
    c[3] = in ? c[0] : INT_MIN; c[4] = in ? c[1] : INT_MIN; c[5] = in ? c[2] : INT_MIN;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < 6; ++j)
    {
        const int r = j < 3 ? __reduce_min_sync(0xffffffffu, c[j]) : __reduce_max_sync(0xffffffffu, c[j]);
        if (lane == 0) part[j][warp] = r;
    }
    __syncthreads();
    if (threadIdx.x < 6)
    {
        const int j = threadIdx.x;
        int r = part[j][0];
        for (int w = 1; w < kThreads / 32; ++w) r = j < 3 ? min(r, part[j][w]) : max(r, part[j][w]);
        if (j < 3) atomicMin(box + j, r); else atomicMax(box + j, r);
    }
}

__global__ void __launch_bounds__(kThreads) k_render_bounds(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y,
                                                            const int32_t* __restrict__ z, int* box)
{
    rd_bounds(n, x, y, z, nullptr, box);
}

// The box of the fusion volume's voxels with weight > 0
__global__ void __launch_bounds__(kThreads) k_live_bounds(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y,
                                                          const int32_t* __restrict__ z, const float* __restrict__ w, int* box)
{
    rd_bounds(n, x, y, z, w, box);
}

struct BrickBox { int lo[3], dim[3]; };

// w: only the voxels with weight > 0 set their brick (nullptr: all)
__device__ __forceinline__ void rd_bricks(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z,
                                          const float* __restrict__ w, const BrickBox& bb, uint32_t* __restrict__ bits)
{
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (v >= n) return;
    if (w && !(w[v] > 0.0f)) return;
    const int bx = (x[v] - bb.lo[0]) >> 3, by = (y[v] - bb.lo[1]) >> 3, bz = (z[v] - bb.lo[2]) >> 3;
    const int64_t idx = (static_cast<int64_t>(bz) * bb.dim[1] + by) * bb.dim[0] + bx;
    atomicOr(bits + (idx >> 5), 1u << (idx & 31));
}

__global__ void k_render_bricks(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z, BrickBox bb,
                                uint32_t* __restrict__ bits)
{
    rd_bricks(n, x, y, z, nullptr, bb, bits);
}

__global__ void k_live_bricks(int64_t n, const int32_t* __restrict__ x, const int32_t* __restrict__ y, const int32_t* __restrict__ z,
                              const float* __restrict__ w, BrickBox bb, uint32_t* __restrict__ bits)
{
    rd_bricks(n, x, y, z, w, bb, bits);
}

} // namespace i3d
