/*
 * i3d_track.h — the frame-to-model tracker (i3d_track.cuh, DESIGN.md §6n), compiled with the renderer whose march it uses for the prediction
 * in i3d_render.cu: the tracker's types and scratch, and the call the engine (i3d_engine.cu) makes with the grid it builds and its stream.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>

#include "i3d_frames.h"
#include "i3d_fusion.h"
#include "i3d_render.h"

namespace i3d
{

// per-pixel / per-tile / per-frame values of one system: 21 upper-triangle entries of J^T J (row by row), 6 of J^T r, r^2, rows
constexpr int kTrackVals = 29;
constexpr int kTrackTile = 16;                  // 16 x 16 pixels per block of k_track_rows
constexpr int kTrackMaxLevels = 4;
// k_track_local_norm (DESIGN.md §6r): 32 x 8 pixels per block; the radius is at most I3D_TRACK_MAX_NORM_RADIUS (its shared rows)
constexpr int kTrackLniTileW = 32, kTrackLniTileH = 8;
constexpr int kTrackLniMaxRadius = I3D_TRACK_MAX_NORM_RADIUS;

// Per-frame state of a call, device-resident: the pose T_cw (camera -> world, double R row-major | t), its float copy for the rows, the
// world -> camera pose returned to the caller, and the outcome.  Written only by k_track_init and k_track_solve.
struct TrackState
{
    double T[12];
    double w2c[12];
    float Tf[12];
    int status, iterations, frozen, pad;
    long long correspondences;
    double residual_sq, update_norm;
};

// A pinhole camera in float (the store's depth camera at one pyramid level)
struct TrackCam { int W, H; float fx, fy, cx, cy; };

// One rows launch: level `cam` of the chunk's frames [gridDim.z]; frame z reads depth / nrm + z * W * H, the prediction planes of the
// chunk (camera pcam, level 0) and its input pose rt_in + 12 * ids[z] (float world -> camera, as the march used it).
struct TrackRows
{
    TrackCam cam, pcam;
    const float* depth; const float* nrm;                 // level planes [n][H][W], [n][H][W][3]
    const float* pdepth; const float* pnrm;               // prediction [n][H0][W0], [n][H0][W0][3]
    const int32_t* ids; const float* rt_in;
    const TrackState* state;                              // the chunk's frames
    float max_dist_sq, min_cos;
    int use_cos;
    uint8_t* mask;                                        // level 0: [n][H0][W0] correspondence mask, else nullptr
    double* partials;                                     // [n][tiles][kTrackVals]
    int tiles_x, tiles_y;
};

// One photometric rows launch (DESIGN.md §6p): level `cam` of the chunk's frames [gridDim.z]; pixel (u, v) samples the prediction pixel
// (step u, step v), step = 2^l, of the level-0 prediction depth / model intensity, and frame z reads the level's intensity, gradient and
// depth planes + z * W * H.
struct TrackPhoto
{
    TrackCam cam, pcam;
    int step;
    const float* inten; const float* gx; const float* gy; const float* depth;   // level planes [n][H][W]
    const float* pdepth; const float* pint;                                     // prediction [n][H0][W0]
    const int32_t* ids; const float* rt_in;
    const TrackState* state;
    float max_distance, max_diff, min_grad_sq;
    double* partials;                                     // [n][tiles][kTrackVals]
    int tiles_x, tiles_y;
};

// One reference-model launch (DESIGN.md §6q): level `cam` of the chunk's frames [gridDim.y]; pixel (u, v) of frame z projects the model
// point of prediction pixel (step u, step v) into its reference (float world -> camera ref_rt + 12 z) and samples the reference's level
// planes + z * W * H there; the value (or the quiet NaN) goes to model at the level-0 index of that prediction pixel.
struct TrackRef
{
    TrackCam cam, pcam;
    int step;
    const float* pdepth;                                  // prediction [n][H0][W0]
    const int32_t* ids; const float* rt_in;               // as TrackRows
    const float* ref_rt;                                  // [n][12]
    const float* inten; const float* depth;               // the references' level planes [n][H][W]
    float max_distance;
    float* model;                                         // [n][H0][W0]
};

// Per-frame photometric outcome of a call (k_track_combine): rows and sum r^2 of the first and the last evaluated system
struct TrackColorState
{
    long long first_rows, last_rows;
    double first_sq, last_sq;
    int have_first, pad;
};

// Tracker scratch of an engine (grows only): the per-call state of n frames, and the chunk's prediction, pyramid, normal and mask planes.
// The planes of the last chunk stay for i3d_debug_get_track_planes.  With a photometric term also the model intensity, the frame
// intensity pyramid with its gradients (i3d_debug_get_track_color_planes), the photometric systems and the combined ones.
struct TrackScratch
{
    Dev<float> rt; Dev<int32_t> ids; Dev<double> pose_in; Dev<TrackState> state;
    Dev<double> sys, sums, partials, rd_partials, rd_sums; Dev<unsigned long long> counters;
    Dev<float> pdepth, pnrm, depth[kTrackMaxLevels], nrm[kTrackMaxLevels]; Dev<uint8_t> mask;
    Dev<int> live_box; Dev<uint32_t> live_bits;           // box and brick bitmap of the fusion volume in progress, rebuilt per use
    Dev<float> pint, lum_c, inten[kTrackMaxLevels], gx[kTrackMaxLevels], gy[kTrackMaxLevels];
    Dev<double> sys_c, sums_c, sums_comb, partials_c; Dev<TrackColorState> cstate; Dev<int32_t> iota;
    // with a reference model (DESIGN.md §6q): the references' ids and float poses, their intensity and depth pyramids, and the model
    // planes of levels 1.. (level 0 is pint), each in the level-0 layout (i3d_debug_get_track_reference_planes)
    Dev<int32_t> ref_ids; Dev<float> ref_rt, ref_inten[kTrackMaxLevels], ref_depth[kTrackMaxLevels], ref_model[kTrackMaxLevels];
    // with norm_radius > 0 (DESIGN.md §6r): the raw intensity pyramids of the frames and of the references, which k_track_local_norm
    // normalises into inten / ref_inten; at I3D_TRACK_CHUNK frames of 640 x 480 over 3 levels 51.6 MB each
    Dev<float> raw_inten[kTrackMaxLevels], raw_ref_inten[kTrackMaxLevels];
    int n = 0, levels = 0, last_m = 0, W[kTrackMaxLevels] = {}, H[kTrackMaxLevels] = {};
    bool color = false;                                   // the last call had a photometric term
    bool reference = false;                               // ... taken from reference frames
};

// The photometric term of a call: its parameters (validated by the caller), the store whose colour frames it reads, and the per-frame
// outcome (may be nullptr).  With ref_ids (host, validated; nullptr: the voxel model of DESIGN.md §6p) the model intensity of frame k is
// sampled from the stored frame ref_ids[k] at its world -> camera pose ref_pose + 12 k (DESIGN.md §6q).
struct TrackColor
{
    const I3DTrackColorParams* P;
    const SensorStore* ss;
    I3DTrackColorInfo* info;
    const int32_t* ref_ids = nullptr;
    const double* ref_pose = nullptr;
};

namespace track
{
// Tracks the stored frames ids[0..n) (validated by the caller; Wl / Hl: the pyramid sizes) of the store's depth planes store_depth
// [store_F][dc] in passes of I3D_TRACK_CHUNK frames.  Per pass: the prediction (k_render_march at the input poses with the depth camera,
// geometry only; rg is the grid without its voxel box, built in rs when the voxel set changed), the depth pyramid (frames::depthdown on
// the gathered store depth) with its normals, then every Gauss-Newton iteration of every level, coarsest first, with no host
// synchronisation; one read-back at the end.  Writes only ts, rs's voxel box, pose_out [n][12] and info [n].
// col (nullptr: depth only) adds the photometric term of DESIGN.md §6p: the colour march (model intensity), the frame intensity pyramid
// with its gradients timed as "track_color", and per system k_track_photo_rows and k_track_combine before the unchanged solve.
void sensor_frames(TrackScratch& ts, RenderState& rs, Timing& tm, RenderGrid rg, const I3DFusionCamera& dc, const float* store_depth, int store_F,
                   int n, const int32_t* ids, const double* pose_in, const I3DTrackParams& P, const int* Wl, const int* Hl, double* pose_out,
                   I3DTrackInfo* info, cudaStream_t st, const TrackColor* col = nullptr);
// sensor_frames with the prediction marched from the fusion volume in progress (k_render_march_live; fs unchanged) instead of a grid.  The
// box and bitmap of the volume's voxels with weight > 0 are built first, timed as "track_bricks"; skip: march with the bitmap
// (i3d_debug_set_render_skip).  Returns non-zero, having tracked nothing, when no voxel has weight > 0.
int fusion_frames(TrackScratch& ts, const FusionState& fs, bool skip, Timing& tm, const SensorStore& ss, int n, const int32_t* ids,
                  const double* pose_in, const I3DTrackParams& P, const int* Wl, const int* Hl, double* pose_out, I3DTrackInfo* info, cudaStream_t st,
                  const TrackColor* col = nullptr);
// Dense frame-to-model odometry over the stored frames ids[0..n) (validated by the caller; repeats allowed), in list order.  Per frame:
// the guess (pose_first for ids[0] when given, which resets fs's motion state; else constant velocity from it), then with no voxel of
// weight > 0 the frame is integrated at the guess (I3D_TRACK_ANCHORED), otherwise fusion_frames' tracking of that one frame (m = 1) and,
// at status 0 only, fusion::integrate at the tracked pose.  Timed as "odometry" (host wall time of the call), "odometry_predict",
// "odometry_icp" and the fusion phases.  Returns non-zero with the message in `error` when fusion::integrate fails.
// reference (col must be set, its ref_ids nullptr): each frame's model intensity comes from the last frame the loop integrated, at the
// pose it was integrated with (fs.ref_id / fs.ref_T, kept like the motion state); a frame with no such reference is tracked on depth alone.
int odometry(TrackScratch& ts, FusionState& fs, bool skip, Timing& tm, const SensorStore& ss, int n, const int32_t* ids, const double* pose_first,
             const I3DTrackParams& P, const int* Wl, const int* Hl, double* pose_out, I3DTrackInfo* info, std::string& error, cudaStream_t st,
             const TrackColor* col = nullptr, bool reference = false);
// The tracker's pose kernels for one device-resident state, for other modules' point-to-plane problems (the reference-mesh registration,
// i3d_register.cuh).  init: k_track_init of pose_in (device [12]).  step: k_tile_sums<kTrackVals> of the partials [blocks][kTrackVals]
// into sums, then k_track_solve of that system (solve = 0: recorded only), its copy into sys and its rows added to *rows.
void pose_init(const double* pose_in, TrackState* state, cudaStream_t st);
void pose_step(int blocks, const double* partials, double* sums, TrackState* state, double* sys, int min_corr, int solve, unsigned long long* rows,
               cudaStream_t st);
} // namespace track

} // namespace i3d
