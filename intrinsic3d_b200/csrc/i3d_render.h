/*
 * i3d_render.h — host interface of the keyframe renderer (i3d_render.cuh, compiled in i3d_render.cu; DESIGN.md §6m).  The kernels live
 * in a device module of their own, so the engine's module holds exactly the kernels of the refinement path; the engine (i3d_engine.cu)
 * owns the buffers and calls these wrappers on its stream.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "i3d_grid.cuh"

namespace i3d
{

// statistic partials per tile and per view: num_hit, num_observed, depth_count, photo_count, depth_abs, depth_sq, photo_abs, photo_sq
constexpr int kRenderStats = 8;
constexpr int kRenderTile = 16;                 // 16 x 16 pixels per block
constexpr int kUndistortIters = 10;             // fixed-point iterations of the inverse lens distortion
// Last lattice index a ray may sample (float(k) is exact up to here).  Never reached by a finite ray: voxel coordinates lie in the
// +-2^20 range of the device hash, so the box diagonal spans fewer than 7.3 M samples of voxel_size / 2.
constexpr int kRenderMaxLattice = 1 << 24;
// Views of one i3d_render_keyframes call: they go in gridDim.z
constexpr int kRenderMaxViews = 65535;

// The grid as the march reads it: g.sdf is the source the surface is cut from, g.sh / sh_has the per-voxel SH (nullptr without
// photometric outputs).  lo / hi: the axis-aligned box of the voxel set in metres (min / max voxel coordinate * voxel_size).
// bricks: bit per 8^3 brick of voxel coordinates, brick (bx, by, bz) = ((X - blo[0]) >> 3, ...), bit (bz * bdim[1] + by) * bdim[0] + bx
// set when the brick holds a voxel; nullptr = march every lattice sample.
struct RenderGrid
{
    GridView g;
    const unsigned long long* keys; const int32_t* vals; uint64_t mask;
    const uint8_t* sh_has;
    float lo[3], hi[3];
    const uint32_t* bricks;
    int blo[3], bdim[3];
};

// The camera of the frame scans (the engine's select_cam): intrinsics * pyr_scale and the distortion, in float
struct RenderCam { float fx, fy, cx, cy; float d[5]; int dist_zero; };

// One batch of views: view z renders frame ids[z] with Rt + 12 * ids[z] (R row-major | t, world -> camera) and compares it with that
// frame's depth / luminance.  Plane pointers are nullptr when not requested; partials [n][tiles][kRenderStats].
struct RenderViews
{
    int n, W, H, tiles_x, tiles_y;
    const int32_t* ids;
    const float* Rt;
    const float* depth; const float* lum;
    float* out_depth; float* out_normal; float* out_albedo; float* out_shading; float* out_intensity;
    double* partials;
    unsigned long long* samples;       // lattice samples evaluated (integer atomics)
    int photometric;
};

namespace render
{
// 1. the bounding box of the voxel coordinates: box[0..2] = min (atomicMin), box[3..5] = max; box must hold INT_MAX / INT_MIN on entry
void bounds(int64_t n, const int32_t* x, const int32_t* y, const int32_t* z, int* box, cudaStream_t st);
// 2. the brick bitmap (zeroed by the caller)
void bricks(int64_t n, const int32_t* x, const int32_t* y, const int32_t* z, const int blo[3], const int bdim[3], uint32_t* bits, cudaStream_t st);
// 3. one thread per pixel, views in gridDim.z: the requested planes and the per-tile statistic partials
void march(const RenderGrid& rg, const RenderCam& cam, const RenderViews& rv, cudaStream_t st);
// 4. out[n][kRenderStats] = the fixed-order sums of the partials of each view
void finish(int n, int tiles, const double* partials, double* out, cudaStream_t st);
} // namespace render

} // namespace i3d
