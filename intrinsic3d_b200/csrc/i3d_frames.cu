/*
 * i3d_frames.cu — keyframe scores, the sensor store and the RGB-D frame store with its pyramid: their kernels (i3d_frames.cuh) and the
 * host code that sequences them (i3d_frames.h).
 */
#include <algorithm>

#include "../../include/i3d_c_api.h"
#include "i3d_frames.cuh"
#include "i3d_frames.h"

namespace i3d
{
namespace
{
// The tiles of a W x H frame's blur partial sums
dim3 blur_tiles(int W, int H) { return dim3((W + kBlurTileW - 1) / kBlurTileW, (H + kBlurTileH - 1) / kBlurTileH); }

// The chunk of F frames scored per pass; sizes ks.partials for it
int score_chunk(ScoreScratch& ks, int F, int W, int H)
{
    const dim3 t = blur_tiles(W, H);
    const int chunk = std::min<int>(F, I3D_KEYFRAME_CHUNK);
    ks.partials.ensure(static_cast<size_t>(chunk) * t.x * t.y * 4);
    return chunk;
}

// Blur scores of the n frames bgr [n][H][W][3] into scores [n]: k_blur_partials into ks.partials, then k_blur_finish
void blur_scores(ScoreScratch& ks, int n, int W, int H, const uint8_t* bgr, double* scores, cudaStream_t st)
{
    const dim3 t = blur_tiles(W, H);
    k_blur_partials<<<dim3(t.x, t.y, n), dim3(32, 8), 0, st>>>(n, W, H, bgr, ks.partials.p);
    k_blur_finish<<<(n + 3) / 4, 128, 0, st>>>(n, static_cast<int>(t.x * t.y), ks.partials.p, scores);
}
} // namespace

void frames::depthdown(int n, int W, int H, const float* src, float* dst, cudaStream_t st)
{
    const dim3 grid((W / 2 + 31) / 32, (H / 2 + 7) / 8, std::min(n, 65535));
    k_frames_depthdown<<<grid, dim3(32, 8), 0, st>>>(n, W, H, src, dst);
}

void frames::pyrdown(int n, int W, int H, const float* src, float* dst, cudaStream_t st)
{
    const int wd = W / 2, hd = H / 2;
    k_frames_pyrdown<<<dim3((wd + 31) / 32, (hd + 7) / 8, std::min(n, 65535)), dim3(32, 8), 0, st>>>(n, W, H, src, dst);
}

void frames::sensor_intensity(const SensorStore& ss, int n, const int32_t* ids, const int32_t* iota, Dev<float>& tmp, float* dst, cudaStream_t st)
{
    const I3DFusionCamera &dc = ss.dcam, &cc = ss.ccam;
    const size_t cpx = static_cast<size_t>(cc.width) * cc.height;
    const bool same = dc.width == cc.width && dc.height == cc.height;
    if (!same) tmp.ensure(cpx * n);
    float* lum = same ? dst : tmp.p;
    for (int k = 0; k < n; ++k)
        k_frames_lum0<<<blocks_for(cpx), kThreads, 0, st>>>(cpx, ss.bgr.p + 3 * cpx * ids[k], lum + cpx * k);
    if (same) return;
    const ResizeCams rc{cc.width, cc.height, cc.fx, cc.fy, cc.cx, cc.cy, dc.width, dc.height, dc.fx, dc.fy, dc.cx, dc.cy};
    k_resize_depth<<<dim3((dc.width + 31) / 32, (dc.height + 7) / 8, std::min(n, 65535)), dim3(32, 8), 0, st>>>(n, iota, rc, tmp.p, dst);
}

void frames::keyframe_scores(ScoreScratch& ks, Timing& tm, int F, int W, int H, const uint8_t* bgr, double* scores, cudaStream_t st)
{
    const size_t img = static_cast<size_t>(W) * H * 3;
    const int chunk = score_chunk(ks, F, W, H);
    ks.bgr.ensure(img * chunk); ks.scores.ensure(chunk);
    begin_timing(tm, {"keyframe_scores", "keyframe_chunks"});
    for (int f0 = 0; f0 < F; f0 += chunk)
    {
        const int n = std::min(chunk, F - f0);
        CK(cudaMemcpyAsync(ks.bgr.p, bgr + img * f0, img * n, cudaMemcpyHostToDevice, st));
        {
            Timer t(tm, st, "keyframe_scores");
            blur_scores(ks, n, W, H, ks.bgr.p, ks.scores.p, st);
        }
        CK(cudaMemcpyAsync(scores + f0, ks.scores.p, n * sizeof(double), cudaMemcpyDeviceToHost, st));
        collect_kernel_times(tm, st);               // synchronises: the chunk buffer is free again
        CK(cudaGetLastError());
        tm.phases["keyframe_chunks"].count += 1;
    }
}

void frames::sensor_keyframe_scores(ScoreScratch& ks, Timing& tm, const SensorStore& ss, double* scores, cudaStream_t st)
{
    const int W = ss.ccam.width, H = ss.ccam.height, F = ss.F;
    const size_t img = static_cast<size_t>(W) * H * 3;
    const int chunk = score_chunk(ks, F, W, H);
    ks.scores.ensure(F);
    begin_timing(tm, {"keyframe_scores", "keyframe_chunks"});
    {
        // the chunks share the partials buffer in stream order: no host synchronisation between them
        Timer t(tm, st, "keyframe_scores");
        for (int f0 = 0; f0 < F; f0 += chunk)
        {
            const int n = std::min(chunk, F - f0);
            blur_scores(ks, n, W, H, ss.bgr.p + img * f0, ks.scores.p + f0, st);
            tm.phases["keyframe_chunks"].count += 1;
        }
    }
    CK(cudaMemcpyAsync(scores, ks.scores.p, F * sizeof(double), cudaMemcpyDeviceToHost, st));
    collect_kernel_times(tm, st);
    CK(cudaGetLastError());
}

void frames::sensor_begin(SensorStore& ss, const I3DFusionCamera& dc, const I3DFusionCamera& cc, int capacity)
{
    const size_t dimg = static_cast<size_t>(dc.width) * dc.height;
    const size_t cimg = static_cast<size_t>(cc.width) * cc.height * 3;
    ss.depth.ensure(dimg * capacity); ss.bgr.ensure(cimg * capacity);
    ss.dcam = dc; ss.ccam = cc; ss.cap = capacity;
}

void frames::sensor_add(SensorStore& ss, int F, const float* depth, const uint8_t* bgr, cudaStream_t st)
{
    const size_t dimg = static_cast<size_t>(ss.dcam.width) * ss.dcam.height;
    const size_t cimg = static_cast<size_t>(ss.ccam.width) * ss.ccam.height * 3;
    CK(cudaMemcpyAsync(ss.depth.p + dimg * ss.F, depth, dimg * F * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ss.bgr.p + cimg * ss.F, bgr, cimg * F, cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    ss.F += F;
}

void frames::select(RgbdStore& rs, Timing& tm, SensorStore& ss, int n, const int32_t* ids, cudaStream_t st)
{
    const I3DFusionCamera &dc = ss.dcam, &cc = ss.ccam;
    const int W = cc.width, H = cc.height;
    const size_t cnt = static_cast<size_t>(n) * W * H, dimg = static_cast<size_t>(dc.width) * dc.height, cimg = static_cast<size_t>(W) * H * 3;
    rs.lum.ensure(cnt); rs.depth.ensure(cnt); rs.bgr.ensure(3 * cnt);
    begin_timing(tm, {"sensor_select", "resize_depth"});
    {
        Timer t(tm, st, "sensor_select");
        for (int k = 0; k < n; ++k)
            CK(cudaMemcpyAsync(rs.bgr.p + cimg * k, ss.bgr.p + cimg * ids[k], cimg, cudaMemcpyDeviceToDevice, st));
        if (dc.width == W && dc.height == H)
        {
            // resizeDepth returns the plane unchanged when the sizes agree, whatever the intrinsics (Q51)
            for (int k = 0; k < n; ++k)
                CK(cudaMemcpyAsync(rs.depth.p + dimg * k, ss.depth.p + dimg * ids[k], dimg * sizeof(float), cudaMemcpyDeviceToDevice, st));
        }
        else
        {
            ss.ids.ensure(n);
            CK(cudaMemcpyAsync(ss.ids.p, ids, n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
            const ResizeCams rc{dc.width, dc.height, dc.fx, dc.fy, dc.cx, dc.cy, W, H, cc.fx, cc.fy, cc.cx, cc.cy};
            Timer tr(tm, st, "resize_depth");
            k_resize_depth<<<dim3((W + 31) / 32, (H + 7) / 8, std::min(n, 65535)), dim3(32, 8), 0, st>>>(n, ss.ids.p, rc, ss.depth.p, rs.depth.p);
        }
        k_frames_lum0<<<blocks_for(cnt), kThreads, 0, st>>>(cnt, rs.bgr.p, rs.lum.p);
    }
    collect_kernel_times(tm, st);
    CK(cudaGetLastError());
    rs.F = n; rs.W = W; rs.H = H;
}

void frames::upload(RgbdStore& rs, int F, int W, int H, const uint8_t* bgr, const float* depth, const float* lum, cudaStream_t st)
{
    const size_t cnt = static_cast<size_t>(F) * W * H;
    rs.lum.ensure(cnt); rs.depth.ensure(cnt); rs.bgr.ensure(3 * cnt);
    CK(cudaMemcpyAsync(rs.bgr.p, bgr, 3 * cnt, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(rs.depth.p, depth, cnt * sizeof(float), cudaMemcpyHostToDevice, st));
    if (lum) CK(cudaMemcpyAsync(rs.lum.p, lum, cnt * sizeof(float), cudaMemcpyHostToDevice, st));
    else k_frames_lum0<<<blocks_for(cnt), kThreads, 0, st>>>(cnt, rs.bgr.p, rs.lum.p);
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    rs.F = F; rs.W = W; rs.H = H;
}

void frames::level(RgbdStore& rs, Timing& tm, int lvl, float* lum, float* depth, cudaStream_t st)
{
    const int F = rs.F;
    Timer t(tm, st, "frames_level");
    if (lvl == 0)
    {
        const size_t cnt = static_cast<size_t>(F) * rs.W * rs.H;
        CK(cudaMemcpyAsync(lum, rs.lum.p, cnt * sizeof(float), cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(depth, rs.depth.p, cnt * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return;
    }
    // the chain level 0 -> 1 -> ... -> lvl, intermediate levels in two ping-pong pairs, the last one straight into lum / depth
    const float* sl = rs.lum.p; const float* sd = rs.depth.p;
    int w = rs.W, h = rs.H;
    for (int k = 1; k <= lvl; ++k)
    {
        const int wd = w / 2, hd = h / 2;
        float* dl = lum; float* dd = depth;
        if (k < lvl)
        {
            const size_t c = static_cast<size_t>(F) * wd * hd;
            rs.tmp[k & 1].ensure(c); rs.tmp[2 + (k & 1)].ensure(c);
            dl = rs.tmp[k & 1].p; dd = rs.tmp[2 + (k & 1)].p;
        }
        pyrdown(F, w, h, sl, dl, st);
        depthdown(F, w, h, sd, dd, st);
        sl = dl; sd = dd; w = wd; h = hd;
    }
}

} // namespace i3d
