/*
 * i3d_recolor.cuh — voxel recolouring on the device (SURVEY.md §8 f2).
 *
 * Replaces Intrinsic3D::recomputeColors (libintrinsic3d/src/refinement/intrinsic3d.cpp:381-409), i.e.
 * SDFColorization::add for every frame + SDFColorization::compute (src/sdf/colorization.cpp:113-189), with
 * computeObservation / computeWeight / filter / computeColor (:215-370) and interpolateRGB (src/rgbd/processing.cpp:236-302).
 *
 * One thread per voxel that has a forward-difference normal.  The frame scan is the one of k_select_obs (the observation weight,
 * the conservative per-warp frame culling and the top-K of i3d_observe.cuh); the best K (weight, frame) keys stay in registers.  The reference keeps a
 * std::vector of observations per voxel (N x F VertexObservation objects across the F add() calls); here nothing is stored:
 * the <= K winning frames are re-projected at the end and their colours fetched bilinearly.
 *
 * Float summation order is the reference's: when the top-K filter runs (more than K observations) the colours are summed in
 * ascending (weight, frame) order (the order std::sort leaves them in; ties broken by frame id, the canonical choice of
 * oracle.cpp), otherwise (K == 0 or at most K observations) in frame order.
 */
#pragma once
#include "i3d_observe.cuh"

namespace i3d
{

// K == 0: no filter (all observations, frame order).  counts[0] += voxels recoloured, counts[1] += observations with weight > 0.
template <int KMAX>
__global__ void __launch_bounds__(kThreads)
k_recolor(GridView g, FrameView fr, const uint8_t* __restrict__ bgr /* [F][H][W][3] */, const float* __restrict__ Rt, SelectCam cam, CullView cull, int K,
          uchar4* __restrict__ rgb_out, unsigned long long* __restrict__ counts)
{
    extern __shared__ float s_rt[];     // [F][12]
    for (int i = threadIdx.x; i < 12 * fr.F; i += blockDim.x) s_rt[i] = Rt[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    float nrm[3] = {0.0f, 0.0f, 0.0f};
    float pt[3] = {0.0f, 0.0f, 0.0f};
    const bool in_range = v < g.n && iso_point(g, v, nrm, pt);     // add(): voxels without a normal collect nothing
    if (__ballot_sync(0xffffffffu, in_range) == 0u) return;
    const int nwords = (fr.F + 31) / 32;
    __shared__ unsigned s_mask[kThreads / 32][kCullMaxWords];
    unsigned* wmask = s_mask[threadIdx.x >> 5];
    const bool culling = frame_candidates(pt, in_range, s_rt, fr, cam, cull, wmask);
    const size_t img = static_cast<size_t>(fr.W) * fr.H;
    const float scale_color = FD(1.0f, 255.0f);
    unsigned long long best[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; ++k) best[k] = 0ull;
    int n_obs = 0;
    float c3[3] = {0.0f, 0.0f, 0.0f}, wsum = 0.0f;
    auto add_color = [&](int f, float wf, const ObsProbe& p) {     // p: the frame's probe, for the sub-pixel position
        const uint8_t* cimg = bgr + img * f * 3;
        const float ws = FM(wf, scale_color);
        c3[0] = FA(c3[0], FM(static_cast<float>(interp_u8(cimg, fr.W, fr.H, p.pu, p.pv, 2)), ws));
        c3[1] = FA(c3[1], FM(static_cast<float>(interp_u8(cimg, fr.W, fr.H, p.pu, p.pv, 1)), ws));
        c3[2] = FA(c3[2], FM(static_cast<float>(interp_u8(cimg, fr.W, fr.H, p.pu, p.pv, 0)), ws));
        wsum = FA(wsum, wf);
    };
#pragma unroll 1
    for (int j = 0; j < nwords; ++j)
    {
        unsigned m = culling ? wmask[j] : 0xffffffffu;
#pragma unroll 1
        while (m)
        {
            const int f = 32 * j + __ffs(m) - 1;
            m &= m - 1;
            if (f >= fr.F) continue;
            const ObsProbe p = obs_probe(pt, s_rt + 12 * f, cam, fr.depth + img * f, fr.W, fr.H);
            const float wf = obs_finish(p, nrm, s_rt + 12 * f, cam);
            if (wf > 0.0f && in_range)
            {
                ++n_obs;
                if (K == 0) add_color(f, wf, p);
                else topk_insert(best, wf, f);
            }
        }
    }
    // per-warp totals -> two atomics
    {
        const unsigned long long col = __popc(__ballot_sync(0xffffffffu, n_obs > 0));
        unsigned long long tot = static_cast<unsigned long long>(n_obs);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
        if (lane == 0 && counts) { atomicAdd(counts, col); atomicAdd(counts + 1, tot); }
    }
    if (n_obs == 0) return;                                  // compute(): no observation => colour unchanged
    if (K > 0)
    {
        // order the kept observations the way computeColor will meet them, then one (non-unrolled) colour loop
        int sel_f[KMAX]; float sel_w[KMAX];
        topk_summation_order(best, n_obs, K, sel_f, sel_w);
#pragma unroll 1
        for (int k = 0; k < KMAX; ++k)
            if (sel_f[k] >= 0) add_color(sel_f[k], sel_w[k], obs_probe(pt, s_rt + 12 * sel_f[k], cam, fr.depth + img * sel_f[k], fr.W, fr.H));
    }
    // computeColor (colorization.cpp:318-354): mean colour, cast<unsigned char> truncates
    if (wsum > 0.0f) { const float s = FD(255.0f, wsum); c3[0] = FM(c3[0], s); c3[1] = FM(c3[1], s); c3[2] = FM(c3[2], s); }
    uchar4 o4 = rgb_out[v];
    o4.x = static_cast<unsigned char>(__float2int_rz(c3[0])); o4.y = static_cast<unsigned char>(__float2int_rz(c3[1])); o4.z = static_cast<unsigned char>(__float2int_rz(c3[2]));
    rgb_out[v] = o4;
}

__global__ void k_interleave_rgb(int64_t n, const uchar4* __restrict__ rgb, uint8_t* __restrict__ out3)
{
    const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    const uchar4 c = rgb[i];
    out3[3 * i] = c.x; out3[3 * i + 1] = c.y; out3[3 * i + 2] = c.z;
}

} // namespace i3d
