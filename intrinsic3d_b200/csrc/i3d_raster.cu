/*
 * i3d_raster.cu — the rasterizer of the resident mesh: its kernels (i3d_raster.cuh) and the host code that sequences them
 * (i3d_raster.h).  Keeping them out of i3d_engine.cu leaves the engine's device module as it is.
 */
#include <vector>

#include "i3d_raster.cuh"

namespace i3d
{
namespace raster
{

void run(RasterState& rs, Timing& tm, const RastMesh& m, const RenderCam& cam, const RastCall& c, I3DRasterStats* stats, I3DRasterInfo* info,
         cudaStream_t st)
{
    const int n = c.n, W = c.W, H = c.H;
    const size_t img = static_cast<size_t>(W) * H, all = static_cast<size_t>(n) * img;
    const int TX = (W + kRastTile - 1) / kRastTile, TY = (H + kRastTile - 1) / kRastTile;
    const int SX = (W + kRenderTile - 1) / kRenderTile, SY = (H + kRenderTile - 1) / kRenderTile;
    int64_t views = std::min<int64_t>(kRastMaxBatchPixels / static_cast<int64_t>(img), kRenderMaxViews);
    if (rs.max_batch > 0) views = std::min<int64_t>(views, rs.max_batch);
    const int batch = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(n, views)));
    // Every allocation comes before the previous planes are touched: a plane buffer that must grow is allocated fresh and swapped in
    // only when all of them and the scratch exist, so a call that runs out of memory leaves the previous planes as they were.
    Dev<float> depth, bary, normal; Dev<int32_t> face; Dev<uint8_t> rgb;
    auto fresh = [](auto& live, auto& f, size_t count) { if (count > live.cap) f.ensure(count); };
    if (c.planes & I3D_RASTER_DEPTH) fresh(rs.depth, depth, all);
    if (c.planes & I3D_RASTER_FACE) fresh(rs.face, face, all);
    if (c.planes & I3D_RASTER_BARY) fresh(rs.bary, bary, 2 * all);
    if (c.planes & I3D_RASTER_NORMAL) fresh(rs.normal, normal, 3 * all);
    if (c.planes & I3D_RASTER_RGB) fresh(rs.rgb, rgb, 3 * all);
    rs.rays.ensure(2 * img); rs.tbox.ensure(4 * static_cast<size_t>(TX) * TY); rs.bands.ensure(2 * static_cast<size_t>(TX + TY));
    rs.keys.ensure(static_cast<size_t>(batch) * img);
    rs.partials.ensure(static_cast<size_t>(batch) * SX * SY * kRastSums);
    rs.sums.ensure(static_cast<size_t>(n) * kRastSums);
    rs.counts.ensure(static_cast<size_t>(n) * kRastCounts); rs.counters.ensure(4);
    if (c.ids) rs.ids.ensure(n);
    begin_timing(tm, {"raster", "raster_bin", "raster_faces", "raster_shade", "raster_tests"});
    rs.have = false;
    if (depth.p) rs.depth.swap(depth);
    if (face.p) rs.face.swap(face);
    if (bary.p) rs.bary.swap(bary);
    if (normal.p) rs.normal.swap(normal);
    if (rgb.p) rs.rgb.swap(rgb);
    if (c.ids) CK(cudaMemcpyAsync(rs.ids.p, c.ids, n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(rs.counts.p, 0, static_cast<size_t>(n) * kRastCounts * sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(rs.counters.p, 0, 4 * sizeof(unsigned long long), st));
    float2* rays = reinterpret_cast<float2*>(rs.rays.p);
    float4* tbox = reinterpret_cast<float4*>(rs.tbox.p);
    float2* rowband = reinterpret_cast<float2*>(rs.bands.p);
    float2* colband = rowband + TY;
    const int32_t* ids = c.ids ? rs.ids.p : nullptr;
    {
        Timer total(tm, st, "raster");
        {
            Timer t(tm, st, "raster_bin");
            k_rast_rays<<<blocks_for(img), kThreads, 0, st>>>(cam, W, H, rays);
            k_rast_tiles<<<blocks_for(static_cast<size_t>(TX) * TY), kThreads, 0, st>>>(W, H, TX, TY, rays, tbox);
            k_rast_band_raw<<<TX + TY, 32, 0, st>>>(TX, TY, tbox, rowband, colband);
            k_rast_bands<<<1, 32, 0, st>>>(TX, TY, rowband, colband);
        }
        for (int v0 = 0; v0 < n; v0 += batch)
        {
            const int nb = std::min(batch, n - v0);
            CK(cudaMemsetAsync(rs.keys.p, 0xFF, static_cast<size_t>(nb) * img * sizeof(unsigned long long), st));
            {
                Timer t(tm, st, "raster_faces");
                const RastBin rb{v0, W, H, TX, TY, ids, c.Rt, rays, tbox, rowband, colband, rs.keys.p, rs.binning ? 1 : 0, rs.counters.p};
                k_rast_faces<<<dim3(blocks_for(static_cast<size_t>(m.F)), nb), kThreads, 0, st>>>(m, rb);
            }
            {
                Timer t(tm, st, "raster_shade");
                RastShade sh{};
                sh.v0 = v0; sh.W = W; sh.H = H; sh.ids = ids; sh.Rt = c.Rt; sh.keys = rs.keys.p; sh.rays = rays;
                sh.depth = c.stats ? c.depth : nullptr; sh.bgr = c.stats ? c.bgr : nullptr; sh.color_source = c.color_source;
                sh.out_depth = (c.planes & I3D_RASTER_DEPTH) ? rs.depth.p : nullptr;
                sh.out_face = (c.planes & I3D_RASTER_FACE) ? rs.face.p : nullptr;
                sh.out_bary = (c.planes & I3D_RASTER_BARY) ? rs.bary.p : nullptr;
                sh.out_normal = (c.planes & I3D_RASTER_NORMAL) ? rs.normal.p : nullptr;
                sh.out_rgb = (c.planes & I3D_RASTER_RGB) ? rs.rgb.p : nullptr;
                sh.partials = rs.partials.p; sh.counts = rs.counts.p;
                k_rast_shade<<<dim3(SX, SY, nb), dim3(kRenderTile, kRenderTile), 0, st>>>(m, sh);
                k_rast_sums<<<blocks_for(static_cast<size_t>(nb) * kRastSums), kThreads, 0, st>>>(nb, SX * SY, rs.partials.p,
                                                                                                   rs.sums.p + static_cast<size_t>(v0) * kRastSums);
            }
        }
    }
    std::vector<double> sums(static_cast<size_t>(n) * kRastSums);
    std::vector<unsigned long long> counts(static_cast<size_t>(n) * kRastCounts);
    unsigned long long counters[4] = {0, 0, 0, 0};
    CK(cudaMemcpyAsync(sums.data(), rs.sums.p, sums.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(counts.data(), rs.counts.p, counts.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(counters, rs.counters.p, sizeof(counters), cudaMemcpyDeviceToHost, st));
    collect_kernel_times(tm, st);
    CK(cudaGetLastError());
    tm.phases["raster_tests"].count = static_cast<int64_t>(counters[3]);
    if (stats && c.stats)
        for (int i = 0; i < n; ++i)
        {
            const unsigned long long* k = counts.data() + static_cast<size_t>(i) * kRastCounts;
            I3DRasterStats s{};
            s.num_covered = static_cast<int64_t>(k[0]); s.num_observed = static_cast<int64_t>(k[1]);
            s.depth_count = static_cast<int64_t>(k[2]); s.color_count = static_cast<int64_t>(k[3]);
            s.depth_abs = sums[static_cast<size_t>(i) * kRastSums]; s.depth_sq = sums[static_cast<size_t>(i) * kRastSums + 1];
            for (int j = 0; j < 3; ++j) { s.color_abs[j] = static_cast<int64_t>(k[4 + j]); s.color_sq[j] = static_cast<int64_t>(k[7 + j]); }
            stats[i] = s;
        }
    if (info)
    {
        I3DRasterInfo inf{};
        inf.num_views = n; inf.num_faces = m.F;
        inf.num_pairs = static_cast<int64_t>(counters[0]); inf.num_straddling = static_cast<int64_t>(counters[1]);
        inf.num_behind = static_cast<int64_t>(counters[2]); inf.num_tests = static_cast<int64_t>(counters[3]);
        for (int i = 0; i < n; ++i) inf.num_covered += static_cast<int64_t>(counts[static_cast<size_t>(i) * kRastCounts]);
        inf.ms_rays = tm.phases["raster_bin"].ms; inf.ms_faces = tm.phases["raster_faces"].ms; inf.ms_shade = tm.phases["raster_shade"].ms;
        *info = inf;
    }
    rs.have = true; rs.keyframes = c.stats; rs.n = n; rs.W = W; rs.H = H; rs.planes = c.planes;
}

} // namespace raster
} // namespace i3d
