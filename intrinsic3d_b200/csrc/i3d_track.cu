/*
 * i3d_track.cu — the frame-to-model tracker's kernels (i3d_track.cuh), compiled as a translation unit of their own, and the host wrappers of
 * i3d_track.h that launch them.  Keeping them out of i3d_engine.cu leaves the engine's device module as it is.
 */
#include "i3d_track.cuh"

namespace i3d
{
namespace track
{
namespace
{
inline unsigned blocks(int64_t n, int threads = kThreads) { return static_cast<unsigned>((n + threads - 1) / threads); }
} // namespace

void init(int n, const double* pose_in, TrackState* state, cudaStream_t st)
{
    k_track_init<<<blocks(n, 64), 64, 0, st>>>(n, pose_in, state);
}

void gather(int n, int W, int H, const int32_t* ids, const float* src, float* dst, cudaStream_t st)
{
    k_track_gather<<<dim3(blocks(static_cast<int64_t>(W) * H), n), kThreads, 0, st>>>(n, W, H, ids, src, dst);
}

void normals(int n, const TrackCam& cam, const float* depth, float* nrm, cudaStream_t st)
{
    k_track_normals<<<dim3(blocks(static_cast<int64_t>(cam.W) * cam.H), n), kThreads, 0, st>>>(cam, depth, nrm);
}

void rows(int n, const TrackRows& tr, cudaStream_t st)
{
    k_track_rows<<<dim3(tr.tiles_x, tr.tiles_y, n), dim3(kTrackTile, kTrackTile), 0, st>>>(tr);
}

void finish(int n, int tiles, const double* partials, double* sums, cudaStream_t st)
{
    k_track_finish<<<blocks(static_cast<int64_t>(n) * kTrackVals), kThreads, 0, st>>>(n, tiles, partials, sums);
}

void solve(int n, const double* sums, TrackState* state, double* sys, int min_corr, int solve, unsigned long long* rows, cudaStream_t st)
{
    k_track_solve<<<blocks(n, 64), 64, 0, st>>>(n, sums, state, sys, min_corr, solve, rows);
}

} // namespace track
} // namespace i3d
