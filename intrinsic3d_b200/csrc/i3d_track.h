/*
 * i3d_track.h — host interface of the frame-to-model tracker (i3d_track.cuh, compiled in i3d_track.cu; DESIGN.md §6n).  The kernels live
 * in a device module of their own, so the engine's module holds exactly the kernels of the refinement path; the engine (i3d_engine.cu)
 * owns the buffers, renders the prediction with render::march and builds the depth pyramid with k_frames_depthdown, and calls these
 * wrappers on its stream.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace i3d
{

// per-pixel / per-tile / per-frame values of one system: 21 upper-triangle entries of J^T J (row by row), 6 of J^T r, r^2, rows
constexpr int kTrackVals = 29;
constexpr int kTrackTile = 16;                  // 16 x 16 pixels per block of k_track_rows
constexpr int kTrackMaxLevels = 4;

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

namespace track
{
// T_cw, its float copy and w2c from the input poses pose_in [n][12] (world -> camera); status and counts cleared
void init(int n, const double* pose_in, TrackState* state, cudaStream_t st);
// dst[k] = the stored depth plane ids[k] (W x H each)
void gather(int n, int W, int H, const int32_t* ids, const float* src, float* dst, cudaStream_t st);
// camera-frame normals of n depth planes by the computeNormals(K, depth, 0.3) rule of k_fuse_normals
void normals(int n, const TrackCam& cam, const float* depth, float* nrm, cudaStream_t st);
// per-tile partials of the chunk's systems at one level
void rows(int n, const TrackRows& tr, cudaStream_t st);
// sums[n][kTrackVals] = the fixed-order sums of each frame's partials
void finish(int n, int tiles, const double* partials, double* sums, cudaStream_t st);
// solve = 1: record, factor, solve and update every frame that is not frozen; 0: record the system only.  sys[n][kTrackVals] gets the
// recorded sums; rows counts the recorded rows (integer atomics)
void solve(int n, const double* sums, TrackState* state, double* sys, int min_corr, int solve, unsigned long long* rows, cudaStream_t st);
} // namespace track

} // namespace i3d
