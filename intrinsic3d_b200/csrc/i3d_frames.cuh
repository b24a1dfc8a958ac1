/*
 * i3d_frames.cuh — keyframe blur scores and the RGB-D image pyramid on the device (DESIGN.md §6i).
 *
 * Restates (paths relative to libintrinsic3d/):
 *   k_blur_partials + k_blur_finish   KeyframeSelection::estimateBlur / estimateBlurCrete    src/keyframe_selection.cpp:219-310
 *   k_frames_lum0                     Pyramid::create's BGR -> float intensity (level 0)     src/rgbd/pyramid.cpp:68-71
 *   k_frames_pyrdown                  Pyramid::downsample (cv::pyrDown, REFLECT_101)         :108-113
 *   k_frames_depthdown                Pyramid::downsampleDepth (masked 2x2 mean)             :116-141
 *   k_resize_depth                    resizeDepth + interpolate<float> (DESIGN.md §6l)        src/rgbd/processing.cpp:129-183, 236-291
 *
 * Every float operation is written with FM/FA/FS/FD (no contraction), in the order tests/frames_ref.py restates, so that a numpy float32
 * restatement reproduces every plane bit for bit.  Equality with a particular OpenCV build is not claimed (it may use FMA or IPP).
 * The blur score's four plane sums are double sums of exactly converted floats in a fixed order: per thread, a fixed warp-shuffle tree,
 * the 8 warps in order, then per frame a fixed-order pass over the tiles.  No atomics: a frame's score depends only on its own pixels.
 */
#pragma once
#include "i3d_grid.cuh"

namespace i3d
{

constexpr int kBlurTileW = 32, kBlurTileH = 32;            // output pixels per block; 32 x 8 threads, 4 rows each
constexpr int kBlurHalo = 5;                                 // +-4 taps, plus the row / column before the tile (backward difference)
constexpr int kBlurSW = kBlurTileW + 2 * kBlurHalo - 1;      // shared tile: rows / columns [t0 - 5, t0 + 36)
constexpr int kBlurSH = kBlurTileH + 2 * kBlurHalo - 1;

// BORDER_REFLECT_101 with one reflection, clamped so that halo cells no output reads stay inside the image
__device__ __forceinline__ int frames_reflect(int i, int n)
{
    i = i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i);
    return min(max(i, 0), n - 1);
}

// OpenCV's fixed-point 8-bit BGR2GRAY, then convertTo(CV_32F, 1/255)
__device__ __forceinline__ float frames_grey(const uint8_t* p)
{
    const int u8 = (1868 * p[0] + 9617 * p[1] + 4899 * p[2] + 8192) >> 14;
    return FM(static_cast<float>(u8), static_cast<float>(1.0 / 255.0));
}

// s = s + w * x[k], k = 0..8, w = float(1/9)
__device__ __forceinline__ float frames_box9(const float* p, int step)
{
    const float w = static_cast<float>(1.0 / 9.0);
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < 9; ++k) s = FA(s, FM(w, p[k * step]));
    return s;
}

__device__ __forceinline__ float frames_relu(float v) { return v > 0.0f ? v : 0.0f; }

// One block per 32x32 tile of one frame: the grey tile with its halo in shared memory, then per output pixel the forward differences of
// the image and of the two box-filtered images (computed on the fly from the tile), their variations, and four double sums per block:
// partials[(f * tiles + tile) * 4 + {s_f_ver, s_v_ver, s_f_hor, s_v_hor}].  Frames f of the chunk: blockIdx.z + k * gridDim.z.
__global__ void __launch_bounds__(256) k_blur_partials(int F, int W, int H, const uint8_t* __restrict__ bgr, double* __restrict__ partials)
{
    __shared__ float g[kBlurSH][kBlurSW];
    __shared__ double warp_sums[8][4];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;
    const int x0 = blockIdx.x * kBlurTileW, y0 = blockIdx.y * kBlurTileH;
    const int tiles = gridDim.x * gridDim.y, tile = blockIdx.y * gridDim.x + blockIdx.x;
    for (int f = blockIdx.z; f < F; f += gridDim.z)
    {
        const uint8_t* img = bgr + static_cast<size_t>(f) * W * H * 3;
        __syncthreads();                                 // the previous frame's reads of g are done
        for (int i = tid; i < kBlurSH * kBlurSW; i += 256)
        {
            const int r = i / kBlurSW, c = i - r * kBlurSW;
            const int gy = frames_reflect(y0 - kBlurHalo + r, H), gx = frames_reflect(x0 - kBlurHalo + c, W);
            g[r][c] = frames_grey(img + (static_cast<size_t>(gy) * W + gx) * 3);
        }
        __syncthreads();
        double s[4] = {0.0, 0.0, 0.0, 0.0};
        const int x = x0 + tx, lx = tx + kBlurHalo;
#pragma unroll
        for (int k = 0; k < 4; ++k)
        {
            const int y = y0 + ty + 8 * k, ly = ty + 8 * k + kBlurHalo;
            if (x >= W || y >= H) continue;
            if (y >= 1)
            {
                const float df = fabsf(FS(g[ly][lx], g[ly - 1][lx]));
                const float db = fabsf(FS(frames_box9(&g[ly - 4][lx], kBlurSW), frames_box9(&g[ly - 5][lx], kBlurSW)));
                s[0] += static_cast<double>(df);
                s[1] += static_cast<double>(frames_relu(FS(df, db)));
            }
            if (x >= 1)
            {
                const float df = fabsf(FS(g[ly][lx], g[ly][lx - 1]));
                const float db = fabsf(FS(frames_box9(&g[ly][lx - 4], 1), frames_box9(&g[ly][lx - 5], 1)));
                s[2] += static_cast<double>(df);
                s[3] += static_cast<double>(frames_relu(FS(df, db)));
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
        {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s[j] += __shfl_down_sync(0xFFFFFFFFu, s[j], o);
        }
        if (tx == 0)
        {
#pragma unroll
            for (int j = 0; j < 4; ++j) warp_sums[ty][j] = s[j];
        }
        __syncthreads();
        if (tid < 4)
        {
            double t = 0.0;
            for (int w = 0; w < 8; ++w) t += warp_sums[w][tid];
            partials[(static_cast<size_t>(f) * tiles + tile) * 4 + tid] = t;
        }
    }
}

// One warp per frame: lane l sums tiles l, l + 32, ... in order, then a fixed shuffle tree; score = 1 - std::max(b_ver, b_hor) with
// b = (s_f - s_v) / s_f, NaN kept as the reference keeps it (std::max(a, NaN) = a, std::max(NaN, b) = NaN).
__global__ void k_blur_finish(int F, int tiles, const double* __restrict__ partials, double* __restrict__ scores)
{
    const int f = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (f >= F) return;
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int t = lane; t < tiles; t += 32)
    {
#pragma unroll
        for (int j = 0; j < 4; ++j) s[j] += partials[(static_cast<size_t>(f) * tiles + t) * 4 + j];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s[j] += __shfl_down_sync(0xFFFFFFFFu, s[j], o);
    }
    if (lane == 0)
    {
        const double b_ver = __ddiv_rn(__dsub_rn(s[0], s[1]), s[0]);
        const double b_hor = __ddiv_rn(__dsub_rn(s[2], s[3]), s[2]);
        scores[f] = __dsub_rn(1.0, (b_ver < b_hor) ? b_hor : b_ver);
    }
}

// Level-0 intensity: c = float(u8) * float(1/255) per channel, then (B 0.114 + G 0.587) + R 0.299
__global__ void k_frames_lum0(size_t count, const uint8_t* __restrict__ bgr, float* __restrict__ lum)
{
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const float inv = static_cast<float>(1.0 / 255.0);
    const uint8_t* p = bgr + 3 * i;
    const float b = FM(static_cast<float>(p[0]), inv), g = FM(static_cast<float>(p[1]), inv), r = FM(static_cast<float>(p[2]), inv);
    lum[i] = FA(FA(FM(b, 0.114f), FM(g, 0.587f)), FM(r, 0.299f));
}

// ((6 c + 4 (b + d)) + a) + e
__device__ __forceinline__ float frames_pyr5(float a, float b, float c, float d, float e)
{
    return FA(FA(FA(FM(6.0f, c), FM(4.0f, FA(b, d))), a), e);
}

// cv::pyrDown of every frame, W x H -> (W / 2) x (H / 2): the row pass (stored as float) at the five source rows of the output pixel,
// then the column pass, times 1/256.  Frames: blockIdx.z + k * gridDim.z.
__global__ void __launch_bounds__(256) k_frames_pyrdown(int F, int W, int H, const float* __restrict__ src, float* __restrict__ dst)
{
    const int Wd = W / 2, Hd = H / 2;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= Wd || y >= Hd) return;
    int cx[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) cx[k] = frames_reflect(2 * x - 2 + k, W);
    for (int f = blockIdx.z; f < F; f += gridDim.z)
    {
        const float* s = src + static_cast<size_t>(f) * W * H;
        float r[5];
#pragma unroll
        for (int k = 0; k < 5; ++k)
        {
            const float* row = s + static_cast<size_t>(frames_reflect(2 * y - 2 + k, H)) * W;
            r[k] = frames_pyr5(__ldg(row + cx[0]), __ldg(row + cx[1]), __ldg(row + cx[2]), __ldg(row + cx[3]), __ldg(row + cx[4]));
        }
        dst[static_cast<size_t>(f) * Wd * Hd + static_cast<size_t>(y) * Wd + x] = FM(frames_pyr5(r[0], r[1], r[2], r[3], r[4]), 1.0f / 256.0f);
    }
}

// Pyramid::downsampleDepth of every frame: taps (2y,2x), (2y,2x+1), (2y+1,2x), (2y+1,2x+1) in that order, only taps > 0, sum / float(cnt),
// 0 without a valid tap
__global__ void __launch_bounds__(256) k_frames_depthdown(int F, int W, int H, const float* __restrict__ src, float* __restrict__ dst)
{
    const int Wd = W / 2, Hd = H / 2;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= Wd || y >= Hd) return;
    for (int f = blockIdx.z; f < F; f += gridDim.z)
    {
        const float* s = src + static_cast<size_t>(f) * W * H + static_cast<size_t>(2 * y) * W + 2 * x;
        const float d[4] = {__ldg(s), __ldg(s + 1), __ldg(s + W), __ldg(s + W + 1)};
        float sum = 0.0f;
        int cnt = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (d[k] > 0.0f) { sum = FA(sum, d[k]); ++cnt; }
        dst[static_cast<size_t>(f) * Wd * Hd + static_cast<size_t>(y) * Wd + x] = cnt > 0 ? FD(sum, static_cast<float>(cnt)) : 0.0f;
    }
}

// The two pinhole cameras of resizeDepth: the depth plane's (in) and the colour camera's (out)
struct ResizeCams
{
    int in_w, in_h;
    float in_fx, in_fy, in_cx, in_cy;
    int out_w, out_h;
    float out_fx, out_fy, out_cx, out_cy;
};

// processing.cpp's resizeDepth + interpolate<float> of one output pixel (DESIGN.md §6l).  The tap (int)(u + 0.5) lies in [0, in_w) exactly
// when u + 0.5 is in (-1, in_w): tested on the float, so an out-of-range or NaN coordinate gives 0 without an undefined cast.  A zero-depth
// tap counts with its weight (Q50); a result of 0 is stored as +0, as the reference leaves the pixel of its zero-initialised output.
__device__ __forceinline__ float resize_depth_px(const ResizeCams& c, const float* __restrict__ src, int x, int y)
{
    const float ifx = FD(1.0f, c.out_fx), ify = FD(1.0f, c.out_fy);
    const float u = FA(FM(c.in_fx, FM(FS(static_cast<float>(x), c.out_cx), ifx)), c.in_cx);
    const float v = FA(FM(c.in_fy, FM(FS(static_cast<float>(y), c.out_cy), ify)), c.in_cy);
    const float tu = FA(u, 0.5f), tv = FA(v, 0.5f);
    if (!(tu > -1.0f && tu < static_cast<float>(c.in_w) && tv > -1.0f && tv < static_cast<float>(c.in_h))) return 0.0f;
    const int x0 = static_cast<int>(floorf(u)), y0 = static_cast<int>(floorf(v)), x1 = x0 + 1, y1 = y0 + 1;
    float wx1 = FS(u, static_cast<float>(x0)), wy1 = FS(v, static_cast<float>(y0));
    float wx0 = FS(1.0f, wx1), wy0 = FS(1.0f, wy1);
    if (x0 < 0 || x0 >= c.in_w) wx0 = 0.0f;
    if (x1 < 0 || x1 >= c.in_w) wx1 = 0.0f;
    if (y0 < 0 || y0 >= c.in_h) wy0 = 0.0f;
    if (y1 < 0 || y1 >= c.in_h) wy1 = 0.0f;
    const float w00 = FM(wx0, wy0), w10 = FM(wx1, wy0), w01 = FM(wx0, wy1), w11 = FM(wx1, wy1);
    const float sw = FA(FA(FA(w00, w10), w01), w11);
    float sum = 0.0f;
    if (w00 > 0.0f) sum = FA(sum, FM(__ldg(src + static_cast<size_t>(y0) * c.in_w + x0), w00));
    if (w01 > 0.0f) sum = FA(sum, FM(__ldg(src + static_cast<size_t>(y1) * c.in_w + x0), w01));
    if (w10 > 0.0f) sum = FA(sum, FM(__ldg(src + static_cast<size_t>(y0) * c.in_w + x1), w10));
    if (w11 > 0.0f) sum = FA(sum, FM(__ldg(src + static_cast<size_t>(y1) * c.in_w + x1), w11));
    if (!(sw > 0.0f)) return 0.0f;
    const float d = FD(sum, sw);
    return d == 0.0f ? 0.0f : d;
}

// resizeDepth of the stored depth planes ids[0..n) into dst [n][out_h][out_w] (output frames: blockIdx.z + k * gridDim.z)
__global__ void __launch_bounds__(256) k_resize_depth(int n, const int32_t* __restrict__ ids, ResizeCams c, const float* __restrict__ src,
                                                      float* __restrict__ dst)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= c.out_w || y >= c.out_h) return;
    const size_t in_px = static_cast<size_t>(c.in_w) * c.in_h, out_px = static_cast<size_t>(c.out_w) * c.out_h;
    for (int f = blockIdx.z; f < n; f += gridDim.z)
        dst[static_cast<size_t>(f) * out_px + static_cast<size_t>(y) * c.out_w + x] = resize_depth_px(c, src + static_cast<size_t>(ids[f]) * in_px, x, y);
}

} // namespace i3d
