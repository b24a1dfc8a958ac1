/*
 * i3d_raster.h — the rasterizer of the resident mesh (i3d_raster.cuh, DESIGN.md §6w), compiled in i3d_raster.cu, a device module of its
 * own: its state and the call the engine (i3d_engine.cu) makes after it has validated the call and computed the poses.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/i3d_types.h"
#include "i3d_host.h"
#include "i3d_render.h"

namespace i3d
{

constexpr int kRastTile = 8;                      // binning tiles: 8 x 8 pixels
constexpr int64_t kRastMaxBatchPixels = 1ll << 27;  // (view, pixel) keys of one pass (1 GiB); larger calls run in batches of views
constexpr int kRastCounts = 10;                   // per-view integer statistics (I3DRasterStats order: 4 counts, colour abs[3], sq[3])
constexpr int kRastSums = 2;                      // per-view double statistics: depth abs, depth sq

// The resident mesh and its texture as the rasterizer reads them; tex_rgb = nullptr: no texture
struct RastMesh
{
    int32_t F; const float* vpos; const uint8_t* vcol; const int3* faces;
    const uint8_t* tex_rgb; int tex_W, tex_H, tex_S, tex_cols;
};

// One call: n views of W x H; view z has the pose Rt + 12 * (ids ? ids[z] : z) (R row-major | t, world -> camera).  Keyframes also
// compare with depth [F][H][W] and the colour frames bgr [F][H][W][3] (nullptr: no colour pairs).
struct RastCall
{
    int n, W, H;
    const int32_t* ids;                 // host ids (keyframes) or nullptr (views)
    const float* Rt;                    // device poses
    const float* depth; const uint8_t* bgr;
    int planes, color_source;
    bool stats;
};

// Rasterizer state of an engine: the planes of the last call (they belong to the resident mesh; the engine drops them), scratch that
// only grows, and the binning switch
struct RasterState
{
    bool binning = true;                // i3d_debug_set_raster_binning
    int max_batch = 0;                  // i3d_debug_set_raster_batch: views per pass at most (0 = as many as kRastMaxBatchPixels allows)
    bool have = false, keyframes = false;
    int n = 0, W = 0, H = 0, planes = 0;
    Dev<float> rays; Dev<float> tbox; Dev<float> bands; Dev<unsigned long long> keys;
    Dev<float> rt; Dev<int32_t> ids;
    Dev<float> depth; Dev<int32_t> face; Dev<float> bary, normal; Dev<uint8_t> rgb;
    Dev<double> partials, sums; Dev<unsigned long long> counts, counters;
};

namespace raster
{
// Rasterizes mesh m (F > 0 faces) into the views of c with the camera cam (the caller validated every argument).  The result becomes
// rs's planes; stats [n] (keyframes, may be nullptr) and info (may be nullptr) get the statistics, counts and device times, timed as
// phases "raster", "raster_bin" (ray table and tile boxes), "raster_faces" and "raster_shade"; i3d_phase_count("raster_tests") = the
// ray-triangle tests.
void run(RasterState& rs, Timing& tm, const RastMesh& m, const RenderCam& cam, const RastCall& c, I3DRasterStats* stats, I3DRasterInfo* info,
         cudaStream_t st);
} // namespace raster

} // namespace i3d
