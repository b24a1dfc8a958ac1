/*
 * i3d_texture.cu — the texture bake of the resident mesh: its kernels (i3d_texture.cuh) and the host code that launches them
 * (i3d_texture.h).  Keeping them out of i3d_engine.cu leaves the engine's device module as it is.
 */
#include <cstring>

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

void bake(TextureState& ts, Timing& tm, const TexMesh& m, const TexLayout& L, const FrameView& fr, const uint8_t* bgr, const SelectCam& cam,
          const CullView& cull, int K, I3DTextureInfo* info, cudaStream_t st)
{
    if (!ts.ev_ready) { for (auto& ev : ts.ev) CK(cudaEventCreate(&ev)); ts.ev_ready = true; }
    ts.have = false; ts.intrinsic = false;
    const size_t texels = static_cast<size_t>(L.W) * L.H;
    ts.rgb.ensure(3 * texels); ts.uv.ensure(6 * static_cast<size_t>(m.F)); ts.counts.ensure(5); ts.observed.ensure(texels);
    const size_t smem = 12 * static_cast<size_t>(fr.F) * sizeof(float);
    auto kern = (K <= 5) ? k_tex_bake<5> : k_tex_bake<I3D_MAX_OBS>;
    if (smem > 48 * 1024)
    {
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        CK(cudaFuncSetAttribute(k_tex_observed, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    }
    CK(cudaMemsetAsync(ts.counts.p, 0, 5 * sizeof(unsigned long long), st));
    CK(cudaEventRecord(ts.ev[0], st));
    kern<<<blocks_for(texels), kThreads, smem, st>>>(m, L, fr, bgr, ts.rt.p, cam, cull, K, ts.rgb.p, ts.counts.p);
    k_tex_uv<<<blocks_for(static_cast<size_t>(m.F)), kThreads, 0, st>>>(m.F, L, ts.uv.p);
    CK(cudaEventRecord(ts.ev[1], st));
    // the observation flags of the decomposition, timed apart: ms_bake stays the time of the atlas and the UVs, i3d_phase_ms("texture_observed")
    // is the flags' time
    begin_timing(tm, {"texture_observed"});
    {
        Timer t(tm, st, "texture_observed");
        k_tex_observed<<<blocks_for(texels), kThreads, smem, st>>>(m, L, fr, ts.rt.p, cam, cull, ts.observed.p);
    }
    unsigned long long h[5] = {0, 0, 0, 0, 0};
    CK(cudaMemcpyAsync(h, ts.counts.p, sizeof(h), cudaMemcpyDeviceToHost, st));
    collect_kernel_times(tm, st);
    CK(cudaGetLastError());
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ts.ev[0], ts.ev[1]));
    ts.W = L.W; ts.H = L.H; ts.S = L.S; ts.cols = L.cols; ts.F = m.F;
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

void decompose(TextureState& ts, const TexMesh& m, const ShLight& light, float min_shading, I3DIntrinsicTextureInfo* info, cudaStream_t st)
{
    if (!ts.ev_ready) { for (auto& ev : ts.ev) CK(cudaEventCreate(&ev)); ts.ev_ready = true; }
    const size_t texels = static_cast<size_t>(ts.W) * ts.H;
    ts.albedo.ensure(3 * texels); ts.shading.ensure(texels); ts.dcounts.ensure(3); ts.drange.ensure(6);
    ts.intrinsic = false;
    const TexLayout L{ts.S, ts.cols, ts.H / ts.S, ts.W, ts.H};
    const unsigned range0[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
    CK(cudaMemsetAsync(ts.dcounts.p, 0, 3 * sizeof(unsigned long long), st));
    CK(cudaMemcpyAsync(ts.drange.p, range0, sizeof(range0), cudaMemcpyHostToDevice, st));
    const TexDecompose d{ts.rgb.p, ts.observed.p, light, min_shading, ts.albedo.p, ts.shading.p, ts.dcounts.p, ts.drange.p};
    CK(cudaEventRecord(ts.ev[0], st));
    k_tex_decompose<<<blocks_for(texels), kThreads, 0, st>>>(m, L, d);
    CK(cudaEventRecord(ts.ev[1], st));
    unsigned long long h[3] = {0, 0, 0};
    unsigned r[6];
    CK(cudaMemcpyAsync(h, ts.dcounts.p, sizeof(h), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(r, ts.drange.p, sizeof(r), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ts.ev[0], ts.ev[1]));
    ts.intrinsic = true;
    if (info)
    {
        I3DIntrinsicTextureInfo inf{};
        inf.atlas_width = ts.W; inf.atlas_height = ts.H;
        inf.num_texels_owned = static_cast<int64_t>(h[0]); inf.num_texels_lit = static_cast<int64_t>(h[1]);
        inf.num_texels_unlit = inf.num_texels_owned - inf.num_texels_lit; inf.num_texels_lit_fallback = static_cast<int64_t>(h[2]);
        auto as_float = [](unsigned u) { float f; std::memcpy(&f, &u, sizeof(f)); return f; };
        for (int k = 0; k < 3; ++k)     // no lit texel: both 0
        {
            inf.albedo_min[k] = h[1] ? as_float(r[k]) : 0.0f;
            inf.albedo_max[k] = h[1] ? as_float(r[3 + k]) : 0.0f;
        }
        inf.ms_decompose = ms;
        *info = inf;
    }
}

} // namespace texture
} // namespace i3d
