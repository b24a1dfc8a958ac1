/*
 * i3d_observe.cuh — the observation rules of SDFColorization (libintrinsic3d/src/sdf/colorization.cpp:192-370) that the observation
 * selection (k_select_obs, i3d_kernels.cuh), the recolouring (k_recolor, i3d_recolor.cuh) and the texture bake (k_tex_bake,
 * i3d_texture.cuh) share: the observation weight of a frame at a point, the conservative per-warp frame culling, the top-K of (weight,
 * frame) keys with the order computeColor sums them in, and the bilinear colour lookup.  No kernels.
 */
#pragma once
#include "i3d_grid.cuh"

namespace i3d
{

struct FrameView
{
    int F, W, H;
    const float* lum; const float* depth;
    double pyr_scale;
};

struct SelectCam { float fx, fy, cx, cy; float d[5]; int dist_zero; float occlusion; };

// SDFColorization::computeObservation -> weight (float pipeline, exact rounding; see oracle.cpp observation_weight), split at its one
// dependent load so that k_select_obs can pipeline it: obs_probe() transforms and projects the point and ISSUES the depth tap, obs_finish()
// consumes it.  The weight is obs_finish(obs_probe(...)).  pu, pv: Camera::project's sub-pixel position pt2f, for the colour lookup of
// the recolouring.
struct ObsProbe { float q0, q1, q2, d, pu, pv; int ok; };
__device__ __forceinline__ ObsProbe obs_probe(const float pt[3], const float* __restrict__ Rt, const SelectCam& cam, const float* __restrict__ depth, int W, int H)
{
    ObsProbe o;
    float q[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) q[k] = FA(FA(FA(FM(Rt[3 * k], pt[0]), FM(Rt[3 * k + 1], pt[1])), FM(Rt[3 * k + 2], pt[2])), Rt[9 + k]);
    o.q0 = q[0]; o.q1 = q[1]; o.q2 = q[2]; o.d = 0.0f; o.ok = 0;
    float x = FD(q[0], q[2]);
    float y = FD(q[1], q[2]);
    if (!cam.dist_zero)
    {
        const float r2 = FA(FM(x, x), FM(y, y));
        const float r4 = FM(r2, r2);
        const float r6 = FM(r4, r2);
        const float dc = FA(FA(FA(1.0f, FM(cam.d[0], r2)), FM(cam.d[1], r4)), FM(cam.d[2], r6));
        const float xn = FA(FA(FM(x, dc), FM(FM(FM(2.0f, cam.d[3]), x), y)), FM(cam.d[4], FA(r2, FM(FM(2.0f, x), x))));
        const float yn = FA(FA(FM(y, dc), FM(FM(FM(2.0f, cam.d[4]), xn), y)), FM(cam.d[3], FA(r2, FM(FM(2.0f, y), y))));
        x = xn; y = yn;
    }
    o.pu = FA(FM(cam.fx, x), cam.cx);
    o.pv = FA(FM(cam.fy, y), cam.cy);
    const float pu5 = FA(o.pu, 0.5f), pv5 = FA(o.pv, 0.5f);
    if (!(pu5 > -2147483000.0f && pu5 < 2147483000.0f && pv5 > -2147483000.0f && pv5 < 2147483000.0f)) return o;
    const int iu = __float2int_rz(pu5), iv = __float2int_rz(pv5);
    if (iu < 0 || iu >= W || iv < 0 || iv >= H) return o;
    o.d = __ldg(depth + static_cast<size_t>(iv) * W + iu);
    o.ok = 1;
    return o;
}
__device__ __forceinline__ float obs_finish(const ObsProbe& o, const float nrm[3], const float* __restrict__ Rt, const SelectCam& cam)
{
    if (!o.ok) return 0.0f;
    const float d = o.d;
    const float q[3] = {o.q0, o.q1, o.q2};
    if (cam.occlusion > 0.0f)
    {
        if (!(d > 0.0f)) return 0.0f;
        const float sd = FS(d, q[2]);
        if (!(fabsf(sd) <= cam.occlusion)) return 0.0f;
    }
    if (d <= 0.0f) return 0.0f;
    float nc[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) nc[k] = FA(FA(FM(Rt[3 * k], nrm[0]), FM(Rt[3 * k + 1], nrm[1])), FM(Rt[3 * k + 2], nrm[2]));
    float w_normal = 0.0f;
    if (!(nc[0] == 0.0f && nc[1] == 0.0f && nc[2] == 0.0f))
    {
        const float qn2 = FA(FA(FM(q[0], q[0]), FM(q[1], q[1])), FM(q[2], q[2]));
        float v0 = q[0], v1 = q[1], v2 = q[2];
        if (qn2 > 0.0f) { const float ql = __fsqrt_rn(qn2); v0 = FD(q[0], ql); v1 = FD(q[1], ql); v2 = FD(q[2], ql); }
        const float dt = FA(FA(FM(v0, nc[0]), FM(v1, nc[1])), FM(v2, nc[2]));
        w_normal = FS(1.0f, fabsf(dt));
        w_normal = (1.0f < w_normal) ? 1.0f : w_normal;           // std::min(w_normal, 1.0f)
        w_normal = (w_normal < 0.0f) ? 0.0f : w_normal;           // std::max(.., 0.0f)
        const float div = FA(1.0f, FM(2.0f, w_normal));
        const float rk = FD(1.0f, FM(FM(div, div), div));
        w_normal = (rk < 0.001f) ? 0.001f : rk;
    }
    // depth weight: the reference computes max(1 - (clamp(d) - d_min)/(d_max - d_min), 1.0f), which is exactly 1.0f for
    // every finite d (Q1); w_normal * 1.0f == w_normal bit-for-bit, so the dead arithmetic is skipped.
    return w_normal;
}

// The iso-point x * voxel_size - n * sdf of voxel v (SDFColorization::add), with the voxel's forward-difference normal.  Returns whether
// the voxel has a normal (where it has none, nrm is zero).
__device__ __forceinline__ bool iso_point(const GridView& g, int64_t v, float nrm[3], float pt[3])
{
    const bool has_normal = surface_normal_f(g, v, nrm);
    const float s = static_cast<float>(g.sdf[v]);
    pt[0] = FS(FM(static_cast<float>(g.x[v]), g.voxel_size), FM(nrm[0], s));
    pt[1] = FS(FM(static_cast<float>(g.y[v]), g.voxel_size), FM(nrm[1], s));
    pt[2] = FS(FM(static_cast<float>(g.z[v]), g.voxel_size), FM(nrm[2], s));
    return has_normal;
}

// ---- conservative frame culling of the frame scans ----------------------------------------------------------------------
// Per frame, 32x32-pixel tiles of the depth map: minimum positive depth (+inf if none) and maximum depth, +inf if the tile holds a NaN
// (k_depth_tiles): with the occlusion test off the reference rejects d <= 0 only, so it observes NaN depths.  Built once per
// i3d_upload_frames.  A warp of a frame scan (32 consecutive voxels = a compact spatial cluster when the grid is in a coherent order)
// bounds its iso-points by a sphere and asks, per frame: can ANY point of the sphere pass the reference's tests (pixel inside the image,
// depth not rejected, |d - z| <= occlusion)?  If not, every voxel of the warp has weight exactly 0 for that frame and the exact per-voxel
// computation is skipped.  The result is bit-identical by construction (only provably-zero weights are skipped):
// tests/test_gpu_zz_cull_bound.py fuzzes frame_may_see against the exact weight on the device, and tests/test_gpu_zz_frame_scan.py holds
// both frame scans bit-equal to the oracle and byte-equal to I3D_NO_CULL where the bounds are tight.
constexpr int kCullTile = 32;
constexpr int kCullMaxWords = 16;     // frames / 32 handled by the culling mask (F <= 512); beyond that no culling

struct CullView { const float* tmin; const float* tmax; int enabled; unsigned long long* stats; /* [0] frames visited, [1] frames total (per warp), optional */ };

// true = the frame may see some point of the sphere (centre c, radius rad), false = provably no voxel of the cluster is visible
__device__ __forceinline__ bool frame_may_see(const float c[3], float rad, const float* __restrict__ Rt, const SelectCam& cam, const CullView& cv,
                                              int f, int W, int H)
{
    const float qx = Rt[0] * c[0] + Rt[1] * c[1] + Rt[2] * c[2] + Rt[9];
    const float qy = Rt[3] * c[0] + Rt[4] * c[1] + Rt[5] * c[2] + Rt[10];
    const float qz = Rt[6] * c[0] + Rt[7] * c[1] + Rt[8] * c[2] + Rt[11];
    const float zmin = qz - rad, zmax = qz + rad;
    if (!(zmin > 1e-3f)) return true;                           // sphere touches the camera plane: no claim
    const float iz = 1.0f / qz;
    float xc = qx * iz, yc = qy * iz;
    // |x/z - xc/zc| <= rad (1 + |xc/zc|) / zmin per axis for every point of the sphere
    const float rnx = rad * (1.0f + fabsf(xc)) / zmin, rny = rad * (1.0f + fabsf(yc)) / zmin;
    float lip = 1.0f;
    if (!cam.dist_zero)
    {
        // lens distortion (Camera::project, y' uses the distorted x', Q2): map the centre exactly, bound the footprint growth by a
        // Lipschitz constant of the distortion map over the disk of normalised radius R that contains the footprint
        const float R = sqrtf(xc * xc + yc * yc) + 1.4143f * fmaxf(rnx, rny);
        const float R2 = R * R;
        const float grow = 3.0f * fabsf(cam.d[0]) * R2 + 5.0f * fabsf(cam.d[1]) * R2 * R2 + 7.0f * fabsf(cam.d[2]) * R2 * R2 * R2 +
                           8.0f * (fabsf(cam.d[3]) + fabsf(cam.d[4])) * R;
        lip = 1.0f + 2.0f * grow * (1.0f + 2.0f * fabsf(cam.d[4]) * R);      // generous: the y' term multiplies the x' growth once more
        const float r2 = xc * xc + yc * yc;
        const float dc = 1.0f + cam.d[0] * r2 + cam.d[1] * r2 * r2 + cam.d[2] * r2 * r2 * r2;
        const float xd = xc * dc + 2.0f * cam.d[3] * xc * yc + cam.d[4] * (r2 + 2.0f * xc * xc);
        const float yd = yc * dc + 2.0f * cam.d[4] * xd * yc + cam.d[3] * (r2 + 2.0f * yc * yc);
        xc = xd; yc = yd;
    }
    const float uc = cam.fx * xc + cam.cx, vc = cam.fy * yc + cam.cy;
    // + 2 px for the float pipeline's rounding and the nearest-pixel rounding
    const float ru = cam.fx * 1.4143f * fmaxf(rnx, rny) * lip * 1.001f + 2.0f;
    const float rv = cam.fy * 1.4143f * fmaxf(rnx, rny) * lip * 1.001f + 2.0f;
    if (uc + ru < 0.0f || uc - ru > static_cast<float>(W) || vc + rv < 0.0f || vc - rv > static_cast<float>(H)) return false;   // entirely outside
    const int TW = (W + kCullTile - 1) / kCullTile, TH = (H + kCullTile - 1) / kCullTile;
    const int tx0 = max(0, static_cast<int>(floorf((uc - ru) / kCullTile))), tx1 = min(TW - 1, static_cast<int>(floorf((uc + ru) / kCullTile)));
    const int ty0 = max(0, static_cast<int>(floorf((vc - rv) / kCullTile))), ty1 = min(TH - 1, static_cast<int>(floorf((vc + rv) / kCullTile)));
    if (tx1 - tx0 > 3 || ty1 - ty0 > 3) return true;            // large footprint: do not bother
    float dmin = __int_as_float(0x7f800000), dmax = 0.0f;
    const float* mn = cv.tmin + static_cast<size_t>(f) * TW * TH;
    const float* mx = cv.tmax + static_cast<size_t>(f) * TW * TH;
    for (int ty = ty0; ty <= ty1; ++ty)
        for (int tx = tx0; tx <= tx1; ++tx) { dmin = fminf(dmin, mn[ty * TW + tx]); dmax = fmaxf(dmax, mx[ty * TW + tx]); }
    if (!(dmax > 0.0f)) return false;                           // no positive depth under the footprint: computeWeight returns 0
    if (cam.occlusion > 0.0f)
    {
        const float tol = cam.occlusion * 1.001f + 1e-4f;
        if (zmin > dmax + tol || zmax < dmin - tol) return false;   // |d - z| <= occlusion impossible
    }
    return true;
}

// The candidate frames of the calling warp: the bounding sphere of the iso-points of its in-range lanes, then frame_may_see per frame
// (lane l tests frames l, l+32, ...).  Writes the warp's (F + 31) / 32 mask words to wmask and returns true, or returns false without
// writing when culling is off or there are more than 32 * kCullMaxWords frames (every frame is a candidate).  All 32 lanes must call it.
__device__ __forceinline__ bool frame_candidates(const float pt[3], bool in_range, const float* __restrict__ s_rt /* [F][12] */, const FrameView& fr,
                                                 const SelectCam& cam, const CullView& cull, unsigned* wmask)
{
    const int nwords = (fr.F + 31) / 32;
    const bool culling = cull.enabled && nwords <= kCullMaxWords;
    if (culling)
    {
        const int lane = threadIdx.x & 31;
        const float big = 3.0e38f;
        float lo[3], hi[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { lo[k] = in_range ? pt[k] : big; hi[k] = in_range ? pt[k] : -big; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int k = 0; k < 3; ++k) { lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o)); hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o)); }
        const float c[3] = {0.5f * (lo[0] + hi[0]), 0.5f * (lo[1] + hi[1]), 0.5f * (lo[2] + hi[2])};
        const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        const float rad = 0.5f * sqrtf(dx * dx + dy * dy + dz * dz) * 1.001f + 1e-4f;
#pragma unroll 1
        for (int j = 0; j < nwords; ++j)
        {
            const int f = 32 * j + lane;
            const bool may = (f < fr.F) && frame_may_see(c, rad, s_rt + 12 * f, cam, cull, f, fr.W, fr.H);
            const unsigned m = __ballot_sync(0xffffffffu, may);
            if (lane == 0) wmask[j] = m;
        }
        __syncwarp();
    }
    return culling;
}

// Top-K of the frame scans: the best KMAX (weight, frame) keys in a small sorted register list, key = weight bits << 32 | frame + 1
// (weights are positive, so a larger key is a larger weight; ties -> higher frame id = the canonical top-K of oracle.cpp).  Descending
// insertion; 0 = empty.
template <int KMAX>
__device__ __forceinline__ void topk_insert(unsigned long long (&best)[KMAX], float wf, int f)
{
    unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(wf)) << 32) | static_cast<unsigned>(f + 1);
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
    {
        const unsigned long long hi2 = key > best[k] ? key : best[k];
        const unsigned long long lo2 = key > best[k] ? best[k] : key;
        best[k] = hi2; key = lo2;
    }
}

// The first K entries of a top-K in ascending frame order: re-keyed as (frame + 1) << 32 | weight bits, empty entries and slots from K
// upwards as ~0, which sorts last.
template <int KMAX>
__device__ __forceinline__ void topk_frame_order(unsigned long long (&best)[KMAX], int K)
{
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
    {
        if (k >= K || best[k] == 0ull) best[k] = ~0ull;
        else best[k] = ((best[k] & 0xffffffffull) << 32) | (best[k] >> 32);
    }
#pragma unroll
    for (int i = 0; i < KMAX; ++i)
#pragma unroll
        for (int j = 0; j + 1 < KMAX - i; ++j)
        {
            const unsigned long long lo = best[j] < best[j + 1] ? best[j] : best[j + 1];
            const unsigned long long hi = best[j] < best[j + 1] ? best[j + 1] : best[j];
            best[j] = lo; best[j + 1] = hi;
        }
}

// The kept observations of a top-K (K > 0) in the order computeColor (colorization.cpp:318-354) sums them: when the filter ran (more
// than K observations) ascending (weight, frame) among the K kept ones, otherwise frame order.  sel_f = frame (-1 = empty slot), sel_w
// = its weight.  Consumes `best`.
template <int KMAX>
__device__ __forceinline__ void topk_summation_order(unsigned long long (&best)[KMAX], int n_obs, int K, int (&sel_f)[KMAX], float (&sel_w)[KMAX])
{
    if (n_obs > K)
    {
        // the filter ran: ascending (weight, frame) among the K kept ones == `best` read backwards; re-key as (frame, weight)
#pragma unroll
        for (int k = 0; k < KMAX / 2; ++k) { const unsigned long long t = best[k]; best[k] = best[KMAX - 1 - k]; best[KMAX - 1 - k] = t; }
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
        {
            // after the reversal, entries beyond the best K sit in front: drop them (slot index KMAX-1-k was the rank)
            const bool keep = (KMAX - 1 - k) < K && best[k] != 0ull;
            best[k] = keep ? (((best[k] & 0xffffffffull) << 32) | (best[k] >> 32)) : ~0ull;
        }
    }
    else
    {
        // the filter returned early: frame order.  At most K keys were inserted, so the slots from K upwards are empty already.
        topk_frame_order(best, K);
    }
    // best[] now holds (frame + 1) << 32 | weight bits in summation order, ~0 = empty
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
    {
        sel_f[k] = best[k] == ~0ull ? -1 : static_cast<int>(best[k] >> 32) - 1;
        sel_w[k] = __uint_as_float(static_cast<unsigned>(best[k] & 0xffffffffull));
    }
}

// interpolate<unsigned char> (src/rgbd/processing.cpp:236-291): bilinear on an interleaved B,G,R image, out-of-image taps dropped
__device__ __forceinline__ unsigned char interp_u8(const uint8_t* __restrict__ img, int w, int h, float x, float y, int channel)
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
    if (w00 > 0.0f) sum = FA(sum, FM(static_cast<float>(img[(static_cast<size_t>(y0) * w + x0) * 3 + channel]), w00));
    if (w01 > 0.0f) sum = FA(sum, FM(static_cast<float>(img[(static_cast<size_t>(y1) * w + x0) * 3 + channel]), w01));
    if (w10 > 0.0f) sum = FA(sum, FM(static_cast<float>(img[(static_cast<size_t>(y0) * w + x1) * 3 + channel]), w10));
    if (w11 > 0.0f) sum = FA(sum, FM(static_cast<float>(img[(static_cast<size_t>(y1) * w + x1) * 3 + channel]), w11));
    if (!(sum_w > 0.0f)) return 0;
    return static_cast<unsigned char>(__float2int_rz(FD(sum, sum_w)));
}

} // namespace i3d
