/*
 * i3d_pixel_ray.cuh — the camera ray of a pixel, shared by the renderer's march (i3d_render.cuh) and the rasterizer (i3d_raster.cuh).
 * No kernels.
 */
#pragma once
#include "i3d_render.h"

namespace i3d
{

// Pixel (u, v) (centre at integer coordinates) -> normalised camera coordinates (x, y): the inverse of obs_probe's projection
// (i3d_observe.cuh), with the lens distortion inverted by kUndistortIters fixed-point steps of the forward model.  The camera ray is
// (x, y, 1).
__device__ __forceinline__ void pixel_ray(const RenderCam& cam, int u, int v, float& x, float& y)
{
    const float xd = FD(FS(__int2float_rn(u), cam.cx), cam.fx), yd = FD(FS(__int2float_rn(v), cam.cy), cam.fy);
    x = xd; y = yd;
    if (!cam.dist_zero)
    {
        for (int it = 0; it < kUndistortIters; ++it)
        {
            const float r2 = FA(FM(x, x), FM(y, y));
            const float r4 = FM(r2, r2);
            const float r6 = FM(r4, r2);
            const float dc = FA(FA(FA(1.0f, FM(cam.d[0], r2)), FM(cam.d[1], r4)), FM(cam.d[2], r6));
            const float tx = FA(FM(FM(FM(2.0f, cam.d[3]), x), y), FM(cam.d[4], FA(r2, FM(FM(2.0f, x), x))));
            const float ty = FA(FM(FM(FM(2.0f, cam.d[4]), xd), y), FM(cam.d[3], FA(r2, FM(FM(2.0f, y), y))));    // y' uses the distorted x'
            x = FD(FS(xd, tx), dc);
            y = FD(FS(yd, ty), dc);
        }
    }
}

} // namespace i3d
