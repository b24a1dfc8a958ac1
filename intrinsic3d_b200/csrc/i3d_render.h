/*
 * i3d_render.h — the keyframe renderer (i3d_render.cuh, DESIGN.md §6m), compiled with the tracker that marches its kernel in i3d_render.cu,
 * a device module of its own: the renderer's types and state, and the call the engine (i3d_engine.cu) makes with the grid and camera it
 * builds and its stream.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/i3d_types.h"
#include "i3d_fusion_view.cuh"
#include "i3d_grid.cuh"
#include "i3d_host.h"

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

// The fusion volume in progress as the march reads it (k_render_march_live): the volume, and the box and bitmap of its voxels with
// weight > 0 in RenderGrid's layout.  Built per call by the tracker (i3d_render.cu), never cached in RenderState.
struct LiveGrid
{
    FuseView v;
    float voxel_size;
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

// Renderer state of an engine: the voxel box and brick bitmap of the current voxel set (built on the first render after a change; the
// engine clears box_ready when the voxel set changes), scratch that only grows, and the resident planes of the last render
struct RenderState
{
    bool skip = true;                  // i3d_debug_set_render_skip
    bool box_ready = false, have_bricks = false;
    int box[6] = {}, blo[3] = {}, bdim[3] = {};
    Dev<int> box_d; Dev<uint32_t> bits;
    Dev<float> rt; Dev<int32_t> ids; Dev<double> partials, sums; Dev<unsigned long long> samples;
    Dev<float> depth, normal, albedo, shading, intensity;
    bool have_render = false;
    int n = 0, planes = 0;
};

namespace render
{
// Renders frames ids[0..n) (validated by the caller) of the W x H planes depth / lum with the poses Rt + 12 * id and the camera cam.  rg is
// the grid without its voxel box, which is built here when the voxel set changed; then the march and the fixed-order finish of the
// statistics, timed as phases "render", "render_bricks" and "render_samples".  Writes only rs and stats [n].
void keyframes(RenderState& rs, Timing& tm, RenderGrid rg, const RenderCam& cam, const float* Rt, int n, const int32_t* ids, int W, int H,
               const float* depth, const float* lum, int planes, bool photometric, I3DRenderStats* stats, cudaStream_t st);
} // namespace render

} // namespace i3d
