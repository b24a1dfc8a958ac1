/*
 * i3d_texture.cuh — the texture bake of the resident mesh (DESIGN.md §6t): k_recolor's colour rule applied per texel of a texture atlas
 * instead of per voxel.  Restated in numpy float32 by tests/texture_ref.py.
 *
 * Layout (analytic, no packing search).  Faces 2c and 2c+1 share square cell c of S x S texels (S = texels_per_face in [6, 256]).
 * ncells = ceil(F / 2); cols = the smallest integer with cols^2 >= ncells; rows = ceil(ncells / cols); the atlas is cols S x rows S
 * texels, cell c at column c % cols, row c / cols.  Local texel (i, j) has its centre at (u, v) = (i + 1/2, j + 1/2), v down the image.
 *   face A = 2c:     UV corners (1, 1), (S-3, 1), (1, S-3) for v0, v1, v2; hypotenuse u + v = S - 2; owns the texels with i + j + 1 < S.
 *   face B = 2c + 1: UV corners (S-1, S-1), (3, S-1), (S-1, 3);           hypotenuse u + v = S + 2; owns the texels with i + j + 1 > S.
 * Texels on the midline i + j + 1 = S, the B half of a last odd cell and the padding cells hold 0.
 * Property (tests/test_texture.py): a bilinear lookup at any (u, v) inside a face's UV triangle reads, with non-zero weight, only texels
 * that face owns, all inside its cell.  The taps are floor(u - 1/2) .. floor(u - 1/2) + 1 (and the same in v).  For A, u, v >= 1 puts
 * them at >= 0 and u, v <= S - 3 at <= S - 3; the far pair sums to at most floor(u + 1/2) + floor(v + 1/2) <= u + v + 1 <= S - 1, and
 * reaches S - 1 only when u + 1/2 and v + 1/2 are integers, where its weight is 0.  For B, u, v <= S - 1 puts them at <= S - 1, u, v >= 3
 * at >= 2, and the near pair sums to floor(u - 1/2) + floor(v - 1/2) > u + v - 3 >= S - 1.  So no colour bleeds across a seam and no
 * dilation pass is needed.
 *
 * Texel to point, in this order (FM / FA / FS / FD: one IEEE float operation each, no contraction):
 *   A: a = (u - 1) / (S - 4),     b = (v - 1) / (S - 4);     B: a = (S - 1 - u) / (S - 4),     b = (S - 1 - v) / (S - 4)
 *   a = a < 0 ? 0 : a;  b = b < 0 ? 0 : b;  s = a + b;  if s > 1: a = a / s, b = b / s
 *   w0 = (1 - a) - b;   P = ((w0 v0 + a v1) + b v2) per coordinate
 * The barycentric form, rather than v0 + a (v1 - v0) + b (v2 - v0), makes P exactly v0, v1, v2 at the UV corners.  Every texel an
 * owned lookup can reach, including the ones between a leg or hypotenuse and the cell edge or midline, samples its own face.
 * The normal is n = (v1 - v0) x (v2 - v0), each component (e1[p] e2[q]) - (e1[q] e2[p]), over its length sqrt((n0 n0 + n1 n1) + n2 n2)
 * (__fsqrt_rn); a zero length leaves n = 0, which gives every frame weight 0 (obs_finish), hence the fallback colour.
 *
 * Texel colour: obs_probe / obs_finish at (P, n) for every frame the warp's culling keeps (the texels are enumerated cell-major, row-major
 * inside a cell, so that a warp's points are the one or two faces of one or two adjacent cells), the top-K of (weight, frame), and the
 * colour sum of k_recolor: frame order when K = 0 or at most K observations, ascending (weight, frame) when the filter ran; c += colour
 * (w / 255) per channel, wsum += w, then c (255 / wsum) truncated.  Written R, G, B (channels 2, 1, 0 of the B, G, R frames).
 * Fallback (no observation): per channel trunc(clamp(((w0 c0 + a c1) + b c2) + 1/2, 0, 255)) of the vertex colours c0, c1, c2 at the
 * clamped (a, b) of the texel.
 *
 * UVs (k_tex_uv, one thread per face): corner k at (col S + u_k) / W and 1 - (row S + v_k) / H, W and H the atlas size.
 */
#pragma once
#include "i3d_observe.cuh"
#include "i3d_texture.h"
#include "i3d_texture_layout.cuh"

namespace i3d
{

// Per warp: (observed texels, observations, kept observations, visited texel-frames, total texel-frames) -> counts[0..4].  The
// register bound: 64 holds KMAX = 5 without spills, KMAX = 8 needs 80.
template <int KMAX>
__global__ void __launch_bounds__(kThreads, KMAX <= 5 ? 4 : 2)
k_tex_bake(TexMesh m, TexLayout L, FrameView fr, const uint8_t* __restrict__ bgr /* [F][H][W][3] */, const float* __restrict__ Rt, SelectCam cam,
           CullView cull, int K, uint8_t* __restrict__ atlas /* [H][W][3] */, unsigned long long* __restrict__ counts)
{
    extern __shared__ float s_rt[];     // [F][12]
    for (int i = threadIdx.x; i < 12 * fr.F; i += blockDim.x) s_rt[i] = Rt[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int S = L.S;
    const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    const int64_t total = static_cast<int64_t>(L.cols) * L.rows * S * S;
    int64_t c = 0;
    int i = 0, j = 0, face = -1;
    if (t < total)
    {
        c = t / (S * S);
        const int r = static_cast<int>(t - c * S * S);
        j = r / S; i = r - j * S;
        if (i + j + 1 < S && 2 * c < m.F) face = static_cast<int>(2 * c);
        else if (i + j + 1 > S && 2 * c + 1 < m.F) face = static_cast<int>(2 * c + 1);
    }
    // the texel's byte in the atlas (padding and unused texels of in-range threads get 0)
    uint8_t* const out = atlas + 3 * (t < total ? ((c / L.cols) * S + j) * L.W + (c % L.cols) * S + i : 0);
    const bool in_range = face >= 0;
    if (__ballot_sync(0xffffffffu, in_range) == 0u)
    {
        if (t < total) { out[0] = 0; out[1] = 0; out[2] = 0; }
        return;
    }
    float pt[3] = {0.0f, 0.0f, 0.0f}, nrm[3] = {0.0f, 0.0f, 0.0f};
    if (in_range)
    {
        const int3 fv = m.faces[face];
        float a, b;
        tex_bary(S, face & 1, static_cast<float>(i) + 0.5f, static_cast<float>(j) + 0.5f, a, b);
        const float w0 = FS(FS(1.0f, a), b);
        const float* p0 = m.vpos + 3 * static_cast<size_t>(fv.x);
        const float* p1 = m.vpos + 3 * static_cast<size_t>(fv.y);
        const float* p2 = m.vpos + 3 * static_cast<size_t>(fv.z);
        float e1[3], e2[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            pt[k] = FA(FA(FM(w0, p0[k]), FM(a, p1[k])), FM(b, p2[k]));
            e1[k] = FS(p1[k], p0[k]); e2[k] = FS(p2[k], p0[k]);
        }
        const float n0 = FS(FM(e1[1], e2[2]), FM(e1[2], e2[1]));
        const float n1 = FS(FM(e1[2], e2[0]), FM(e1[0], e2[2]));
        const float n2 = FS(FM(e1[0], e2[1]), FM(e1[1], e2[0]));
        const float len = __fsqrt_rn(FA(FA(FM(n0, n0), FM(n1, n1)), FM(n2, n2)));
        if (len > 0.0f) { nrm[0] = FD(n0, len); nrm[1] = FD(n1, len); nrm[2] = FD(n2, len); }
    }
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
    int visited = 0;
#pragma unroll 1
    for (int jw = 0; jw < nwords; ++jw)
    {
        unsigned mk = culling ? wmask[jw] : 0xffffffffu;
#pragma unroll 1
        while (mk)
        {
            const int f = 32 * jw + __ffs(mk) - 1;
            mk &= mk - 1;
            if (f >= fr.F) continue;
            ++visited;
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
    // per-warp totals -> five atomics
    {
        const unsigned owned = __ballot_sync(0xffffffffu, in_range);
        const unsigned long long observed = __popc(__ballot_sync(0xffffffffu, n_obs > 0));
        unsigned long long tot = static_cast<unsigned long long>(n_obs);
        unsigned long long kept = static_cast<unsigned long long>(K == 0 || n_obs < K ? n_obs : K);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { tot += __shfl_xor_sync(0xffffffffu, tot, o); kept += __shfl_xor_sync(0xffffffffu, kept, o); }
        if (lane == 0)
        {
            const unsigned long long nown = __popc(owned);
            atomicAdd(counts, observed); atomicAdd(counts + 1, tot); atomicAdd(counts + 2, kept);
            atomicAdd(counts + 3, nown * static_cast<unsigned long long>(visited)); atomicAdd(counts + 4, nown * static_cast<unsigned long long>(fr.F));
        }
    }
    if (!in_range)
    {
        if (t < total) { out[0] = 0; out[1] = 0; out[2] = 0; }
        return;
    }
    if (n_obs == 0)
    {
        // no frame observes the texel: the barycentric blend of the face's vertex colours at the texel's (a, b), recomputed here
        const int3 fv = m.faces[face];
        float a, b;
        tex_bary(S, face & 1, static_cast<float>(i) + 0.5f, static_cast<float>(j) + 0.5f, a, b);
        const float w0 = FS(FS(1.0f, a), b);
        const uint8_t* q0 = m.vcol + 3 * static_cast<size_t>(fv.x);
        const uint8_t* q1 = m.vcol + 3 * static_cast<size_t>(fv.y);
        const uint8_t* q2 = m.vcol + 3 * static_cast<size_t>(fv.z);
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            float x = FA(FA(FA(FM(w0, static_cast<float>(q0[k])), FM(a, static_cast<float>(q1[k]))), FM(b, static_cast<float>(q2[k]))), 0.5f);
            x = x < 0.0f ? 0.0f : (x > 255.0f ? 255.0f : x);
            out[k] = static_cast<uint8_t>(__float2int_rz(x));
        }
        return;
    }
    if (K > 0)
    {
        int sel_f[KMAX]; float sel_w[KMAX];
        topk_summation_order(best, n_obs, K, sel_f, sel_w);
#pragma unroll 1
        for (int k = 0; k < KMAX; ++k)
        {
            // slot k by an unrolled select, so that sel_f / sel_w stay in registers (no local memory)
            int f = -1; float wf = 0.0f;
#pragma unroll
            for (int q = 0; q < KMAX; ++q) { f = q == k ? sel_f[q] : f; wf = q == k ? sel_w[q] : wf; }
            if (f >= 0) add_color(f, wf, obs_probe(pt, s_rt + 12 * f, cam, fr.depth + img * f, fr.W, fr.H));
        }
    }
    if (wsum > 0.0f) { const float s = FD(255.0f, wsum); c3[0] = FM(c3[0], s); c3[1] = FM(c3[1], s); c3[2] = FM(c3[2], s); }
    out[0] = static_cast<uint8_t>(__float2int_rz(c3[0])); out[1] = static_cast<uint8_t>(__float2int_rz(c3[1])); out[2] = static_cast<uint8_t>(__float2int_rz(c3[2]));
}

// The per-corner OBJ UVs: uv [F][3][2]
__global__ void k_tex_uv(int32_t F, TexLayout L, float* __restrict__ uv)
{
    const int32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int c = f >> 1;
    const float x0 = static_cast<float>((c % L.cols) * L.S), y0 = static_cast<float>((c / L.cols) * L.S);
    const float W = static_cast<float>(L.W), H = static_cast<float>(L.H);
#pragma unroll
    for (int k = 0; k < 3; ++k)
    {
        float u, v;
        tex_corner(L.S, f & 1, k, u, v);
        uv[6 * static_cast<size_t>(f) + 2 * k] = FD(FA(x0, u), W);
        uv[6 * static_cast<size_t>(f) + 2 * k + 1] = FS(1.0f, FD(FA(y0, v), H));
    }
}

} // namespace i3d
