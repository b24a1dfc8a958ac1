/*
 * i3d_track.cuh — frame-to-model tracking on the device (DESIGN.md §6n): point-to-plane ICP of stored depth frames against the surface
 * rendered at their input poses, over the depth pyramid, with per-frame 6 x 6 normal equations solved in double.
 *
 *   k_track_init     one thread per frame: T_cw = inverse of the input pose, its float copy, the returned pose = the input
 *   k_track_gather   the chunk's stored depth planes side by side (level 0 of its pyramid)
 *   k_track_normals  camera-frame normals by the computeNormals(K, depth, 0.3) rule of k_fuse_normals, frames in gridDim.y
 *   k_track_rows     one thread per pixel, 16 x 16 tiles, frames in gridDim.z: association, gates, the point-to-plane row and its
 *                    29 products, reduced per tile (fixed warp shuffle tree, then the warps in order)
 *   k_tile_sums<kTrackVals> (i3d_render.cuh)  per (frame, value) the frame's tiles summed in order
 *   k_track_solve    one thread per frame: Cholesky of the 6 x 6 system in a fixed order, xi = -A^-1 b, T_cw <- [Rodrigues(w) | v] T_cw
 *
 * The photometric term of the _rgbd calls (DESIGN.md §6p):
 *   k_track_grad        central differences of the frame intensity pyramid, frames in gridDim.y
 *   k_track_photo_rows  one thread per pixel of a level: the model sample at prediction pixel (2^l u, 2^l v), the intensity residual at its
 *                       projection, the gates and the row [g_w x q, -g_w], reduced as k_track_rows reduces
 *   k_track_combine     one thread per frame: A_g + lam^2 A_c, b_g + lam^2 b_c, the geometric r^2 and rows, for the unchanged k_track_solve
 *
 * The reference model of the _ref calls (DESIGN.md §6q), which replaces the voxel colours as k_track_photo_rows' model intensity:
 *   k_track_ref_model   one thread per pixel of a level: the model point of prediction pixel (2^l u, 2^l v) sampled from the frame's
 *                       reference image at the reference's pose, or the quiet NaN
 *
 * The locally normalised intensity of the _ref calls with norm_radius > 0 (DESIGN.md §6r), applied per level to the frame's and the
 * reference's raw intensity pyramids before k_track_grad and k_track_ref_model read them:
 *   k_track_local_norm  one thread per pixel of a level, frames in gridDim.y: (I - mu) / sqrt(var + eps^2) over the clipped window
 *
 * Compiled with the renderer in i3d_render.cu, which launches them (track::sensor_frames, i3d_track.h).  Every float
 * operation is explicitly rounded and every double operation is an explicit __d*_rn (no FMA contraction), so tests/track_ref.py restates
 * the planes, masks and sums exactly.  A frame's bytes depend only on that frame.
 */
#pragma once
#include "i3d_grid.cuh"
#include "i3d_track.h"

namespace i3d
{

#define DM(a, b) __dmul_rn((a), (b))
#define DA(a, b) __dadd_rn((a), (b))
#define DS(a, b) __dsub_rn((a), (b))

// R (row-major 3 x 3) times v, sums left to right, plus t when given
__device__ __forceinline__ void tr_xform(const float* R, const float* t, const float v[3], float out[3])
{
#pragma unroll
    for (int d = 0; d < 3; ++d)
    {
        const float s = FA(FA(FM(R[3 * d], v[0]), FM(R[3 * d + 1], v[1])), FM(R[3 * d + 2], v[2]));
        out[d] = t ? FA(s, t[d]) : s;
    }
}

// world -> camera of T_cw (R | t): R^T | -(R^T t), in double
__device__ __forceinline__ void tr_inverse(const double* T, double* out)
{
#pragma unroll
    for (int i = 0; i < 3; ++i)
    {
#pragma unroll
        for (int j = 0; j < 3; ++j) out[3 * i + j] = T[3 * j + i];
        out[9 + i] = -DA(DA(DM(T[i], T[9]), DM(T[3 + i], T[10])), DM(T[6 + i], T[11]));
    }
}

__global__ void k_track_init(int n, const double* __restrict__ pose_in, TrackState* __restrict__ state)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const double* P = pose_in + 12 * static_cast<int64_t>(k);
    TrackState& s = state[k];
    tr_inverse(P, s.T);                 // the inverse of R | t has the same form: R^T | -(R^T t)
#pragma unroll
    for (int i = 0; i < 12; ++i) { s.w2c[i] = P[i]; s.Tf[i] = __double2float_rn(s.T[i]); }
    s.status = 0; s.iterations = 0; s.frozen = 0; s.pad = 0;
    s.correspondences = 0; s.residual_sq = 0.0; s.update_norm = 0.0;
}

__global__ void k_track_gather(int n, int W, int H, const int32_t* __restrict__ ids, const float* __restrict__ src, float* __restrict__ dst)
{
    const int64_t img = static_cast<int64_t>(W) * H;
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= img) return;
    const int k = blockIdx.y;
    dst[k * img + i] = src[static_cast<int64_t>(ids[k]) * img + i];
}

// The rule of k_fuse_normals (depth_normal) for frame blockIdx.y
__global__ void k_track_normals(TrackCam cam, const float* __restrict__ depth_all, float* __restrict__ nrm_all)
{
    const int64_t img = static_cast<int64_t>(cam.W) * cam.H;
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= img) return;
    const float* depth = depth_all + blockIdx.y * img;
    float* nrm = nrm_all + 3 * blockIdx.y * img;
    const float3 n = depth_normal(depth, cam.W, cam.H, cam.fx, cam.fy, cam.cx, cam.cy, i);
    nrm[3 * i] = n.x; nrm[3 * i + 1] = n.y; nrm[3 * i + 2] = n.z;
}

// The model point of prediction pixel (iu, iv) at depth zm, as the march built the ray of that pixel (camera c0, input pose R0 | t0):
// q = o0 + z_m R0^T (x', y', 1), o0 = -R0^T t0
__device__ __forceinline__ void tr_model_point(const float* R0, const TrackCam& c0, int iu, int iv, float zm, float q[3])
{
    const float xn = FD(FS(__int2float_rn(iu), c0.cx), c0.fx), yn = FD(FS(__int2float_rn(iv), c0.cy), c0.fy);
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        const float o = -FA(FA(FM(R0[k], R0[9]), FM(R0[3 + k], R0[10])), FM(R0[6 + k], R0[11]));
        const float dir = FA(FA(FM(R0[k], xn), FM(R0[3 + k], yn)), R0[6 + k]);
        q[k] = FA(o, FM(zm, dir));
    }
}

// The correspondence of pixel (u, v) of frame z at the current pose (DESIGN.md §6n): p (world), q (model point), n_m (model normal)
__device__ __forceinline__ bool tr_associate(const TrackRows& tr, int z, int u, int v, const float* Tf, float p[3], float q[3], float nm[3])
{
    const int64_t pix = (static_cast<int64_t>(z) * tr.cam.H + v) * tr.cam.W + u;
    const float d = tr.depth[pix];
    if (!(d > 0.0f)) return false;
    const float vc[3] = {FM(FD(FS(__int2float_rn(u), tr.cam.cx), tr.cam.fx), d), FM(FD(FS(__int2float_rn(v), tr.cam.cy), tr.cam.fy), d), d};
    tr_xform(Tf, Tf + 9, vc, p);
    // projection into the prediction (level 0, input pose R0 | t0), pixel int(x + 0.5f) (nv::round, Q35)
    const float* R0 = tr.rt_in + 12 * static_cast<int64_t>(tr.ids[z]);
    float pc[3];
    tr_xform(R0, R0 + 9, p, pc);
    if (!(pc[2] > 0.0f)) return false;
    const TrackCam& c0 = tr.pcam;
    const float tu = FA(FA(FM(c0.fx, FD(pc[0], pc[2])), c0.cx), 0.5f), tv = FA(FA(FM(c0.fy, FD(pc[1], pc[2])), c0.cy), 0.5f);
    if (!(tu > -1.0f && tu < static_cast<float>(c0.W) && tv > -1.0f && tv < static_cast<float>(c0.H))) return false;
    const int iu = __float2int_rz(tu), iv = __float2int_rz(tv);
    const int64_t pp = (static_cast<int64_t>(z) * c0.H + iv) * c0.W + iu;
    const float zm = tr.pdepth[pp];
    if (!(zm > 0.0f)) return false;
    nm[0] = tr.pnrm[3 * pp]; nm[1] = tr.pnrm[3 * pp + 1]; nm[2] = tr.pnrm[3 * pp + 2];
    if (nm[0] == 0.0f && nm[1] == 0.0f && nm[2] == 0.0f) return false;
    tr_model_point(R0, c0, iu, iv, zm, q);
    float dsq = 0.0f;
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        const float e = FS(p[k], q[k]);
        dsq = FA(dsq, FM(e, e));
    }
    if (!(dsq <= tr.max_dist_sq)) return false;
    if (tr.use_cos)
    {
        const float* nc = tr.nrm + 3 * pix;
        float nin[3];
        tr_xform(Tf, nullptr, nc, nin);
        const float dot = FA(FA(FM(nin[0], nm[0]), FM(nin[1], nm[1])), FM(nin[2], nm[2]));
        if (!(dot >= tr.min_cos)) return false;
    }
    return true;
}

// The 29 products of one pixel's row (J, r, cnt), each summed over the warp by a fixed shuffle tree as it is formed (lane 0 keeps the
// warp's sums), then the 8 warps in order into the partials of tile (blockIdx.x, blockIdx.y) of frame z
__device__ __forceinline__ void tr_tile_partials(double (&warp_sums)[kTrackTile * kTrackTile / 32][kTrackVals], const double (&J)[6], double r, double cnt, int tid, int z,
                                                 int tiles_x, int tiles_y, double* partials)
{
    const int lane = tid & 31, warp = tid >> 5;
    int j = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
    {
#pragma unroll
        for (int b = a; b < 6; ++b, ++j)
        {
            double x = DM(J[a], J[b]);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x = DA(x, __shfl_down_sync(0xffffffffu, x, o));
            if (lane == 0) warp_sums[warp][j] = x;
        }
    }
#pragma unroll
    for (int a = 0; a < 8; ++a, ++j)
    {
        double x = a < 6 ? DM(J[a], r) : (a == 6 ? DM(r, r) : cnt);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x = DA(x, __shfl_down_sync(0xffffffffu, x, o));
        if (lane == 0) warp_sums[warp][j] = x;
    }
    __syncthreads();
    if (tid < kTrackVals)
    {
        double t = warp_sums[0][tid];
#pragma unroll
        for (int w = 1; w < kTrackTile * kTrackTile / 32; ++w) t = DA(t, warp_sums[w][tid]);
        const int64_t tile = (static_cast<int64_t>(z) * tiles_y + blockIdx.y) * tiles_x + blockIdx.x;
        partials[tile * kTrackVals + tid] = t;
    }
}

// One thread per pixel of frame blockIdx.z at the rows launch's level
__global__ void __launch_bounds__(kTrackTile * kTrackTile) k_track_rows(TrackRows tr)
{
    __shared__ double warp_sums[kTrackTile * kTrackTile / 32][kTrackVals];
    const int u = blockIdx.x * kTrackTile + threadIdx.x, v = blockIdx.y * kTrackTile + threadIdx.y, z = blockIdx.z;
    const int tid = threadIdx.y * kTrackTile + threadIdx.x;
    const TrackState& s = tr.state[z];
    const bool frozen = s.frozen != 0;
    double J[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, r = 0.0, cnt = 0.0;
    if (u < tr.cam.W && v < tr.cam.H && !frozen)
    {
        float Tf[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) Tf[i] = s.Tf[i];
        float p[3], q[3], nm[3];
        const bool ok = tr_associate(tr, z, u, v, Tf, p, q, nm);
        if (tr.mask) tr.mask[(static_cast<int64_t>(z) * tr.cam.H + v) * tr.cam.W + u] = ok ? 1 : 0;
        if (ok)
        {
            double pd[3], nd[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) { pd[k] = static_cast<double>(p[k]); nd[k] = static_cast<double>(nm[k]); }
            r = DA(DA(DM(nd[0], DS(pd[0], static_cast<double>(q[0]))), DM(nd[1], DS(pd[1], static_cast<double>(q[1])))),
                   DM(nd[2], DS(pd[2], static_cast<double>(q[2]))));
            J[0] = DS(DM(pd[1], nd[2]), DM(pd[2], nd[1]));
            J[1] = DS(DM(pd[2], nd[0]), DM(pd[0], nd[2]));
            J[2] = DS(DM(pd[0], nd[1]), DM(pd[1], nd[0]));
            J[3] = nd[0]; J[4] = nd[1]; J[5] = nd[2];
            cnt = 1.0;
        }
    }
    else if (u < tr.cam.W && v < tr.cam.H && tr.mask)
        tr.mask[(static_cast<int64_t>(z) * tr.cam.H + v) * tr.cam.W + u] = 0;
    tr_tile_partials(warp_sums, J, r, cnt, tid, z, tr.tiles_x, tr.tiles_y, tr.partials);
}

// ---- the photometric term (DESIGN.md §6p) ----------------------------------------------------------------------------------------

// Central differences FM(0.5, I[+1] - I[-1]) of frame blockIdx.y's intensity plane on 1..W-2 x 1..H-2, 0 on the border
__global__ void k_track_grad(TrackCam cam, const float* __restrict__ inten_all, float* __restrict__ gx_all, float* __restrict__ gy_all)
{
    const int64_t img = static_cast<int64_t>(cam.W) * cam.H;
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= img) return;
    const float* I = inten_all + blockIdx.y * img;
    const int y = static_cast<int>(i / cam.W), x = static_cast<int>(i - static_cast<int64_t>(y) * cam.W);
    float gx = 0.0f, gy = 0.0f;
    if (x >= 1 && y >= 1 && x < cam.W - 1 && y < cam.H - 1)
    {
        gx = FM(0.5f, FS(I[i + 1], I[i - 1]));
        gy = FM(0.5f, FS(I[i + cam.W], I[i - cam.W]));
    }
    gx_all[blockIdx.y * img + i] = gx;
    gy_all[blockIdx.y * img + i] = gy;
}

// Bilinear sample of plane P (row stride W) at x0 + fx, y0 + fy: along x, then y
__device__ __forceinline__ float tr_bilinear(const float* __restrict__ P, int W, int x0, int y0, float fx, float fy)
{
    const float* a = P + static_cast<int64_t>(y0) * W + x0;
    const float r0 = FA(a[0], FM(fx, FS(a[1], a[0]))), r1 = FA(a[W], FM(fx, FS(a[W + 1], a[W])));
    return FA(r0, FM(fy, FS(r1, r0)));
}

// The projection of the camera-frame point xc into level camera c, for a bilinear sample there: false unless xc is in front (z > 0),
// all four taps lie in [1, W - 2] x [1, H - 2] (tested on the float: a NaN fails) and the level depth plane's nearest pixel d is not
// occluding (d > 0, |d - z| <= max_distance).  Otherwise the corner (x0, y0) and the fractions (fx, fy) of tr_bilinear.
__device__ __forceinline__ bool tr_project(const TrackCam& c, const float* __restrict__ depth, float max_distance, const float xc[3], int& x0, int& y0,
                                           float& fx, float& fy)
{
    if (!(xc[2] > 0.0f)) return false;
    const float x = FA(FM(c.fx, FD(xc[0], xc[2])), c.cx), y = FA(FM(c.fy, FD(xc[1], xc[2])), c.cy);
    if (!(x >= 1.0f && x < static_cast<float>(c.W - 2) && y >= 1.0f && y < static_cast<float>(c.H - 2))) return false;
    const float d = depth[static_cast<int64_t>(__float2int_rz(FA(y, 0.5f))) * c.W + __float2int_rz(FA(x, 0.5f))];
    if (!(d > 0.0f && fabsf(FS(d, xc[2])) <= max_distance)) return false;
    const float xf = floorf(x), yf = floorf(y);
    x0 = __float2int_rz(xf); y0 = __float2int_rz(yf);
    fx = FS(x, xf); fy = FS(y, yf);
    return true;
}

// One thread per pixel (u, v) of level l of frame blockIdx.z: the model sample at prediction pixel (2^l u, 2^l v), the intensity residual
// at its projection with the current pose, the gates and the photometric row, reduced as k_track_rows reduces (DESIGN.md §6p)
__global__ void __launch_bounds__(kTrackTile * kTrackTile) k_track_photo_rows(TrackPhoto tp)
{
    __shared__ double warp_sums[kTrackTile * kTrackTile / 32][kTrackVals];
    const int u = blockIdx.x * kTrackTile + threadIdx.x, v = blockIdx.y * kTrackTile + threadIdx.y, z = blockIdx.z;
    const int tid = threadIdx.y * kTrackTile + threadIdx.x;
    const TrackState& s = tp.state[z];
    double J[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, r = 0.0, cnt = 0.0;
    if (u < tp.cam.W && v < tp.cam.H && s.frozen == 0)
    {
        const TrackCam& c0 = tp.pcam;
        const int iu = u * tp.step, iv = v * tp.step;
        const int64_t pp = (static_cast<int64_t>(z) * c0.H + iv) * c0.W + iu;
        const float zm = tp.pdepth[pp];
        if (zm > 0.0f)
        {
            float q[3];
            tr_model_point(tp.rt_in + 12 * static_cast<int64_t>(tp.ids[z]), c0, iu, iv, zm, q);
            // x_c = R^T (q - t) with the float camera -> world pose
            float Tf[12];
#pragma unroll
            for (int i = 0; i < 12; ++i) Tf[i] = s.Tf[i];
            const float e[3] = {FS(q[0], Tf[9]), FS(q[1], Tf[10]), FS(q[2], Tf[11])};
            float xc[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) xc[d] = FA(FA(FM(Tf[d], e[0]), FM(Tf[3 + d], e[1])), FM(Tf[6 + d], e[2]));
            const TrackCam& c = tp.cam;
            const int64_t img = static_cast<int64_t>(c.W) * c.H;
            int x0, y0;
            float fx, fy;
            if (tr_project(c, tp.depth + z * img, tp.max_distance, xc, x0, y0, fx, fy))
            {
                const float If = tr_bilinear(tp.inten + z * img, c.W, x0, y0, fx, fy);
                const float gx = tr_bilinear(tp.gx + z * img, c.W, x0, y0, fx, fy);
                const float gy = tr_bilinear(tp.gy + z * img, c.W, x0, y0, fx, fy);
                const float rc = FS(If, tp.pint[pp]);
                if (fabsf(rc) <= tp.max_diff && FA(FM(gx, gx), FM(gy, gy)) >= tp.min_grad_sq)
                {
                    // d r / d x_c, then world: g_w = R g_c; xi perturbs on the left, so J = [g_w x q, -g_w]
                    const float gfx = FM(gx, c.fx), gfy = FM(gy, c.fy);
                    const float gc[3] = {FD(gfx, xc[2]), FD(gfy, xc[2]), -FD(FA(FM(gfx, xc[0]), FM(gfy, xc[1])), FM(xc[2], xc[2]))};
                    float gw[3];
                    tr_xform(Tf, nullptr, gc, gw);
                    double g[3], qd[3];
#pragma unroll
                    for (int k = 0; k < 3; ++k) { g[k] = static_cast<double>(gw[k]); qd[k] = static_cast<double>(q[k]); }
                    J[0] = DS(DM(g[1], qd[2]), DM(g[2], qd[1]));
                    J[1] = DS(DM(g[2], qd[0]), DM(g[0], qd[2]));
                    J[2] = DS(DM(g[0], qd[1]), DM(g[1], qd[0]));
                    J[3] = -g[0]; J[4] = -g[1]; J[5] = -g[2];
                    r = static_cast<double>(rc);
                    cnt = 1.0;
                }
            }
        }
    }
    tr_tile_partials(warp_sums, J, r, cnt, tid, z, tp.tiles_x, tp.tiles_y, tp.partials);
}

// ---- the reference model (DESIGN.md §6q) ---------------------------------------------------------------------------------------------

// One thread per pixel (u, v) of level l of frame blockIdx.y: the model point q of prediction pixel (2^l u, 2^l v), projected into the
// frame's reference and sampled from the reference's level-l intensity, with k_track_photo_rows' bounds and occlusion tests (tr_project)
__global__ void k_track_ref_model(TrackRef tf)
{
    const TrackCam& c = tf.cam;
    const int64_t img = static_cast<int64_t>(c.W) * c.H;
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= img) return;
    const int z = blockIdx.y;
    const int v = static_cast<int>(i / c.W), u = static_cast<int>(i - static_cast<int64_t>(v) * c.W);
    const TrackCam& c0 = tf.pcam;
    const int iu = u * tf.step, iv = v * tf.step;
    const int64_t pp = (static_cast<int64_t>(z) * c0.H + iv) * c0.W + iu;
    // the quiet NaN where any test fails: k_track_photo_rows then forms rc = I_f - NaN = NaN, and its gate fabsf(rc) <= max_diff (an
    // ordered compare, FSETP.LE) is false, so the pixel gives no row
    float val = __int_as_float(0x7FC00000);
    const float zm = tf.pdepth[pp];
    if (zm > 0.0f)
    {
        float q[3];
        tr_model_point(tf.rt_in + 12 * static_cast<int64_t>(tf.ids[z]), c0, iu, iv, zm, q);
        const float* Rr = tf.ref_rt + 12 * static_cast<int64_t>(z);
        float xr[3];
        tr_xform(Rr, Rr + 9, q, xr);
        int x0, y0;
        float fx, fy;
        if (tr_project(c, tf.depth + z * img, tf.max_distance, xr, x0, y0, fx, fy)) val = tr_bilinear(tf.inten + z * img, c.W, x0, y0, fx, fy);
    }
    tf.model[pp] = val;
}

// ---- locally normalised intensity (DESIGN.md §6r) ------------------------------------------------------------------------------------

// One thread per pixel of a kTrackLniTileW x kTrackLniTileH tile (blockIdx.x, row-major over the tiles) of frame blockIdx.y's plane src
// [W x H]: dst = (I - mu) / sqrt(max(m2 - mu^2, 0) + eps^2) over the (2r+1)^2 window clipped to the image, mu = S1 / n, m2 = S2 / n, n the
// float count of its pixels; exactly 0 where the window is constant (its min equals its max).  Separable: the tile's rows with their r
// halo rows are summed along the row (taps in ascending x) into shared memory, then each pixel sums its column of those (ascending y).
__global__ void __launch_bounds__(kTrackLniTileW * kTrackLniTileH) k_track_local_norm(int W, int H, int r, float eps,
                                                                                        const float* __restrict__ src_all, float* __restrict__ dst_all)
{
    constexpr int kRows = kTrackLniTileH + 2 * kTrackLniMaxRadius;
    __shared__ float s1[kRows][kTrackLniTileW], s2[kRows][kTrackLniTileW], mn[kRows][kTrackLniTileW], mx[kRows][kTrackLniTileW];
    const int64_t img = static_cast<int64_t>(W) * H;
    const float* src = src_all + blockIdx.y * img;
    const int tiles_x = (W + kTrackLniTileW - 1) / kTrackLniTileW;
    const int tx = static_cast<int>(blockIdx.x % tiles_x), ty = static_cast<int>(blockIdx.x / tiles_x);
    const int x = tx * kTrackLniTileW + threadIdx.x, y0 = ty * kTrackLniTileH - r, y = y0 + r + threadIdx.y;
    const int xa = max(x - r, 0), xb = min(x + r, W - 1);
    for (int j = threadIdx.y; j < kTrackLniTileH + 2 * r; j += kTrackLniTileH)
    {
        const int yy = y0 + j;
        if (yy < 0 || yy >= H || x >= W) continue;
        const float* row = src + static_cast<int64_t>(yy) * W;
        float a = 0.0f, b = 0.0f, lo = INFINITY, hi = -INFINITY;
        for (int xx = xa; xx <= xb; ++xx)
        {
            const float t = row[xx];
            a = FA(a, t); b = FA(b, FM(t, t)); lo = fminf(lo, t); hi = fmaxf(hi, t);
        }
        s1[j][threadIdx.x] = a; s2[j][threadIdx.x] = b; mn[j][threadIdx.x] = lo; mx[j][threadIdx.x] = hi;
    }
    __syncthreads();
    if (x >= W || y >= H) return;
    const int ya = max(y - r, 0), yb = min(y + r, H - 1);
    float a = 0.0f, b = 0.0f, lo = INFINITY, hi = -INFINITY;
    for (int yy = ya; yy <= yb; ++yy)
    {
        const int j = yy - y0;
        a = FA(a, s1[j][threadIdx.x]); b = FA(b, s2[j][threadIdx.x]); lo = fminf(lo, mn[j][threadIdx.x]); hi = fmaxf(hi, mx[j][threadIdx.x]);
    }
    const int64_t i = static_cast<int64_t>(y) * W + x;
    float out = 0.0f;
    if (lo != hi)
    {
        const float n = __int2float_rn((xb - xa + 1) * (yb - ya + 1));
        const float mu = FD(a, n), m2 = FD(b, n);
        const float var = fmaxf(FS(m2, FM(mu, mu)), 0.0f);
        out = FD(FS(src[i], mu), __fsqrt_rn(FA(var, FM(eps, eps))));
    }
    dst_all[blockIdx.y * img + i] = out;
}

// One thread per frame that is not frozen: the system k_track_solve reads, A = A_g + lam2 A_c and b = b_g + lam2 b_c (entries 0..26;
// exactly the geometric entries for lam2 = 0), with the geometric sum r^2 and row count (27, 28); records the photometric system and
// its rows and sum r^2 (the first and the last evaluated), and adds its rows to *rows.
__global__ void k_track_combine(int n, double lam2, const double* __restrict__ sums_g, const double* __restrict__ sums_c,
                                const TrackState* __restrict__ state, TrackColorState* __restrict__ cstate, double* __restrict__ out,
                                double* __restrict__ sys_c, unsigned long long* rows)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n || state[k].frozen) return;
    const double* G = sums_g + static_cast<int64_t>(k) * kTrackVals;
    const double* P = sums_c + static_cast<int64_t>(k) * kTrackVals;
    double* o = out + static_cast<int64_t>(k) * kTrackVals;
    double* sc = sys_c + static_cast<int64_t>(k) * kTrackVals;
    for (int j = 0; j < 27; ++j) o[j] = lam2 == 0.0 ? G[j] : DA(G[j], DM(lam2, P[j]));
    o[27] = G[27]; o[28] = G[28];
    for (int j = 0; j < kTrackVals; ++j) sc[j] = P[j];
    TrackColorState& cs = cstate[k];
    const long long nr = static_cast<long long>(P[28]);
    if (!cs.have_first) { cs.first_rows = nr; cs.first_sq = P[27]; cs.have_first = 1; }
    cs.last_rows = nr; cs.last_sq = P[27];
    atomicAdd(rows, static_cast<unsigned long long>(nr));
}

// One thread per frame.  Records the system; with solve = 1: freezes on too few rows or a non-finite system, factors A = L L^T
// (j = 0..5: d = A_jj - sum_k<j L_jk^2, in k order; L_jj = sqrt(d), refused unless d > 0; L_ij = (A_ij - sum_k<j L_ik L_jk) / L_jj), solves
// L y = -b, L^T xi = y, and applies T_cw <- [Rodrigues(w) | v] T_cw (xi = (w, v)).
__global__ void k_track_solve(int n, const double* __restrict__ sums, TrackState* __restrict__ state, double* __restrict__ sys, int min_corr,
                              int solve, unsigned long long* rows)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    TrackState& s = state[k];
    if (s.frozen) return;
    const double* S = sums + static_cast<int64_t>(k) * kTrackVals;
    double* out = sys + static_cast<int64_t>(k) * kTrackVals;
    bool finite = true;
    for (int i = 0; i < kTrackVals; ++i) { out[i] = S[i]; finite = finite && isfinite(S[i]); }
    s.correspondences = static_cast<long long>(S[28]);
    s.residual_sq = S[27];
    atomicAdd(rows, static_cast<unsigned long long>(s.correspondences));
    if (!solve) return;
    if (s.correspondences < min_corr) { s.status = 1; s.frozen = 1; return; }
    if (!finite) { s.status = 3; s.frozen = 1; return; }
    double A[6][6], L[6][6], b[6], y[6], x[6];
    int j = 0;
    for (int a = 0; a < 6; ++a)
        for (int c = a; c < 6; ++c, ++j) { A[a][c] = S[j]; A[c][a] = S[j]; }
    for (int a = 0; a < 6; ++a) b[a] = S[21 + a];
    for (int c = 0; c < 6; ++c)
    {
        double d = A[c][c];
        for (int m = 0; m < c; ++m) d = DS(d, DM(L[c][m], L[c][m]));
        if (!(d > 0.0)) { s.status = 2; s.frozen = 1; return; }
        L[c][c] = __dsqrt_rn(d);
        for (int i = c + 1; i < 6; ++i)
        {
            double t = A[i][c];
            for (int m = 0; m < c; ++m) t = DS(t, DM(L[i][m], L[c][m]));
            L[i][c] = __ddiv_rn(t, L[c][c]);
        }
    }
    for (int i = 0; i < 6; ++i)
    {
        double t = -b[i];
        for (int m = 0; m < i; ++m) t = DS(t, DM(L[i][m], y[m]));
        y[i] = __ddiv_rn(t, L[i][i]);
    }
    for (int i = 5; i >= 0; --i)
    {
        double t = y[i];
        for (int m = i + 1; m < 6; ++m) t = DS(t, DM(L[m][i], x[m]));
        x[i] = __ddiv_rn(t, L[i][i]);
    }
    // Rodrigues: R = I + (sin th / th) K + ((1 - cos th) / th^2) K^2, K = [w]x; R = I for th = 0
    const double th2 = DA(DA(DM(x[0], x[0]), DM(x[1], x[1])), DM(x[2], x[2]));
    const double th = __dsqrt_rn(th2);
    double R[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
    if (th > 0.0)
    {
        const double sa = __ddiv_rn(sin(th), th), sb = __ddiv_rn(DS(1.0, cos(th)), th2);
        const double K[9] = {0.0, -x[2], x[1], x[2], 0.0, -x[0], -x[1], x[0], 0.0};
        for (int a = 0; a < 3; ++a)
            for (int c = 0; c < 3; ++c)
            {
                const double k2 = DA(DA(DM(K[3 * a], K[c]), DM(K[3 * a + 1], K[3 + c])), DM(K[3 * a + 2], K[6 + c]));
                R[3 * a + c] = DA(DA(R[3 * a + c], DM(sa, K[3 * a + c])), DM(sb, k2));
            }
    }
    double T[12];
    for (int a = 0; a < 3; ++a)
    {
        for (int c = 0; c < 3; ++c) T[3 * a + c] = DA(DA(DM(R[3 * a], s.T[c]), DM(R[3 * a + 1], s.T[3 + c])), DM(R[3 * a + 2], s.T[6 + c]));
        T[9 + a] = DA(DA(DA(DM(R[3 * a], s.T[9]), DM(R[3 * a + 1], s.T[10])), DM(R[3 * a + 2], s.T[11])), x[3 + a]);
    }
    bool ok = true;
    for (int i = 0; i < 6; ++i) ok = ok && isfinite(x[i]);
    for (int i = 0; i < 12; ++i) ok = ok && isfinite(T[i]);
    if (!ok) { s.status = 3; s.frozen = 1; return; }
    for (int i = 0; i < 12; ++i) { s.T[i] = T[i]; s.Tf[i] = __double2float_rn(T[i]); }
    tr_inverse(T, s.w2c);
    double un = 0.0;
    for (int i = 0; i < 6; ++i) un = DA(un, DM(x[i], x[i]));
    s.update_norm = __dsqrt_rn(un);
    s.iterations += 1;
}

#undef DM
#undef DA
#undef DS

} // namespace i3d
