/*
 * i3d_frames.h — keyframe scores, the sensor store and the RGB-D frame store with its pyramid (i3d_frames.cuh, DESIGN.md §6i, §6l),
 * compiled in i3d_frames.cu, a device module of its own: the stores the engine owns, and the calls the engine (i3d_engine.cu) and the
 * tracker (i3d_render.cu) make with their stream.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/i3d_types.h"
#include "i3d_grid.cuh"
#include "i3d_host.h"

namespace i3d
{

// The sensor store (i3d_sensor_frames_begin / add): the raw sequence, depth [cap][depth cam] in thresholded metres, colour
// [cap][colour cam][3] B,G,R.  Keyframe scores, fusion, i3d_select_rgbd_frames and the tracker read it; only add writes it.
struct SensorStore
{
    int cap = 0, F = 0;
    I3DFusionCamera dcam{}, ccam{};
    Dev<float> depth; Dev<uint8_t> bgr; Dev<int32_t> ids;       // ids: the selection's frame ids on the device
};

// The RGB-D frame store (i3d_upload_rgbd_frames, i3d_select_rgbd_frames): F level-0 keyframes of W x H; i3d_use_rgbd_level builds
// level l from it
struct RgbdStore
{
    int F = 0, W = 0, H = 0;
    Dev<float> lum, depth, tmp[4]; Dev<uint8_t> bgr;            // tmp: intermediate levels, luminance [0..1], depth [2..3]
};

// Keyframe-score scratch: one chunk of host frames, its per-tile partial sums and the scores
struct ScoreScratch
{
    Dev<uint8_t> bgr; Dev<double> partials, scores;
};

namespace frames
{
// Pyramid::downsampleDepth (k_frames_depthdown) of n W x H depth planes into n (W / 2) x (H / 2) planes
void depthdown(int n, int W, int H, const float* src, float* dst, cudaStream_t st);
// cv::pyrDown (k_frames_pyrdown) of n W x H planes into n (W / 2) x (H / 2) planes
void pyrdown(int n, int W, int H, const float* src, float* dst, cudaStream_t st);
// The level-0 intensity of the stored colour frames ids[0..n) (host list, validated by the caller) in the depth camera, into dst
// [n][depth cam]: k_frames_lum0 of each frame's colour plane, then resizeDepth's mapping and interpolate<float> (k_resize_depth) from the
// colour camera to the depth camera with the identity list iota [n] (device: 0, 1, ...).  With equal sizes that is a copy (Q51), so
// lum0 writes dst directly; otherwise tmp holds the colour-size planes.
void sensor_intensity(const SensorStore& ss, int n, const int32_t* ids, const int32_t* iota, Dev<float>& tmp, float* dst, cudaStream_t st);
// Blur scores of F host frames of W x H (validated by the caller), uploaded in chunks of I3D_KEYFRAME_CHUNK: one "keyframe_scores" timer
// per chunk, and a synchronisation per chunk, which frees the chunk buffer again
void keyframe_scores(ScoreScratch& ks, Timing& tm, int F, int W, int H, const uint8_t* bgr, double* scores, cudaStream_t st);
// Blur scores of every frame of the sensor store (validated by the caller) in chunks of I3D_KEYFRAME_CHUNK: one "keyframe_scores" timer
// around all chunks, with no host synchronisation between them
void sensor_keyframe_scores(ScoreScratch& ks, Timing& tm, const SensorStore& ss, double* scores, cudaStream_t st);
// Sizes the sensor store for `capacity` frames of the two cameras (validated by the caller, which has emptied the store)
void sensor_begin(SensorStore& ss, const I3DFusionCamera& dc, const I3DFusionCamera& cc, int capacity);
// Appends F host frames (validated by the caller) to the sensor store
void sensor_add(SensorStore& ss, int F, const float* depth, const uint8_t* bgr, cudaStream_t st);
// The frame store from the sensor frames ids[0..n) (validated by the caller): colour gathered, depth resized to the colour camera
// (resizeDepth; a copy when the sizes agree), level-0 luminance.  Timed as "sensor_select" and "resize_depth".
void select(RgbdStore& rs, Timing& tm, SensorStore& ss, int n, const int32_t* ids, cudaStream_t st);
// The frame store from F host frames of W x H (validated by the caller); lum may be nullptr (computed from bgr)
void upload(RgbdStore& rs, int F, int W, int H, const uint8_t* bgr, const float* depth, const float* lum, cudaStream_t st);
// Level lvl of the frame store (W and H halved lvl times, validated by the caller) into lum / depth, timed as "frames_level": a copy at
// level 0, else the chain 0 -> 1 -> ... -> lvl
void level(RgbdStore& rs, Timing& tm, int lvl, float* lum, float* depth, cudaStream_t st);
} // namespace frames

} // namespace i3d
