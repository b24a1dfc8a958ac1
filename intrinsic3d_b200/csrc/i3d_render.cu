/*
 * i3d_render.cu — the keyframe renderer's kernels (i3d_render.cuh), compiled as a translation unit of their own, and the host wrappers of
 * i3d_render.h that launch them.  Keeping them out of i3d_engine.cu leaves the engine's device module as it is.
 */
#include "i3d_render.cuh"

namespace i3d
{
namespace render
{
namespace
{
inline unsigned blocks(int64_t n) { return static_cast<unsigned>((n + kThreads - 1) / kThreads); }
} // namespace

void bounds(int64_t n, const int32_t* x, const int32_t* y, const int32_t* z, int* box, cudaStream_t st)
{
    k_render_bounds<<<blocks(n), kThreads, 0, st>>>(n, x, y, z, box);
}

void bricks(int64_t n, const int32_t* x, const int32_t* y, const int32_t* z, const int blo[3], const int bdim[3], uint32_t* bits, cudaStream_t st)
{
    const BrickBox bb{{blo[0], blo[1], blo[2]}, {bdim[0], bdim[1], bdim[2]}};
    k_render_bricks<<<blocks(n), kThreads, 0, st>>>(n, x, y, z, bb, bits);
}

void march(const RenderGrid& rg, const RenderCam& cam, const RenderViews& rv, cudaStream_t st)
{
    const dim3 grid(rv.tiles_x, rv.tiles_y, rv.n), block(kRenderTile, kRenderTile);
    k_render_march<<<grid, block, 0, st>>>(rg, cam, rv);
}

void finish(int n, int tiles, const double* partials, double* out, cudaStream_t st)
{
    k_render_finish<<<blocks(static_cast<int64_t>(n) * kRenderStats), kThreads, 0, st>>>(n, tiles, partials, out);
}

} // namespace render
} // namespace i3d
