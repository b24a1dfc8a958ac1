/*
 * i3d_texture.cu — the texture bake of the resident mesh: its kernels (i3d_texture.cuh) and the host code that launches them
 * (i3d_texture.h).  Keeping them out of i3d_engine.cu leaves the engine's device module as it is.
 */
#include "i3d_texture.cuh"

namespace i3d
{
namespace texture
{

bool layout(int64_t F, int S, TexLayout& L)
{
    const int64_t ncells = (F + 1) / 2;
    int64_t cols = 1;
    while (cols * cols < ncells) ++cols;
    const int64_t rows = (ncells + cols - 1) / cols;
    if (cols * S > I3D_TEXTURE_MAX_SIDE || rows * S > I3D_TEXTURE_MAX_SIDE) return false;
    L.S = S; L.cols = static_cast<int>(cols); L.rows = static_cast<int>(rows); L.W = static_cast<int>(cols * S); L.H = static_cast<int>(rows * S);
    return true;
}

void bake(TextureState& ts, const TexMesh& m, const TexLayout& L, const FrameView& fr, const uint8_t* bgr, const SelectCam& cam, const CullView& cull,
          int K, I3DTextureInfo* info, cudaStream_t st)
{
    if (!ts.ev_ready) { for (auto& ev : ts.ev) CK(cudaEventCreate(&ev)); ts.ev_ready = true; }
    ts.have = false;
    const size_t texels = static_cast<size_t>(L.W) * L.H;
    ts.rgb.ensure(3 * texels); ts.uv.ensure(6 * static_cast<size_t>(m.F)); ts.counts.ensure(5);
    const size_t smem = 12 * static_cast<size_t>(fr.F) * sizeof(float);
    auto kern = (K <= 5) ? k_tex_bake<5> : k_tex_bake<I3D_MAX_OBS>;
    if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    CK(cudaMemsetAsync(ts.counts.p, 0, 5 * sizeof(unsigned long long), st));
    CK(cudaEventRecord(ts.ev[0], st));
    kern<<<blocks_for(texels), kThreads, smem, st>>>(m, L, fr, bgr, ts.rt.p, cam, cull, K, ts.rgb.p, ts.counts.p);
    k_tex_uv<<<blocks_for(static_cast<size_t>(m.F)), kThreads, 0, st>>>(m.F, L, ts.uv.p);
    CK(cudaEventRecord(ts.ev[1], st));
    unsigned long long h[5] = {0, 0, 0, 0, 0};
    CK(cudaMemcpyAsync(h, ts.counts.p, sizeof(h), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ts.ev[0], ts.ev[1]));
    ts.W = L.W; ts.H = L.H; ts.F = m.F;
    ts.have = true;
    if (info)
    {
        I3DTextureInfo inf{};
        inf.atlas_width = L.W; inf.atlas_height = L.H; inf.num_faces = m.F;
        inf.num_texels_owned = static_cast<int64_t>(m.F) * L.S * (L.S - 1) / 2;
        inf.num_texels_observed = static_cast<int64_t>(h[0]);
        inf.num_texels_fallback = inf.num_texels_owned - inf.num_texels_observed;
        inf.num_observations = static_cast<int64_t>(h[1]); inf.num_observations_kept = static_cast<int64_t>(h[2]);
        inf.num_texel_frames_visited = static_cast<int64_t>(h[3]); inf.num_texel_frames_total = static_cast<int64_t>(h[4]);
        inf.ms_bake = ms;
        *info = inf;
    }
}

} // namespace texture
} // namespace i3d
