/*
 * i3d_texture.h — the texture bake of the resident mesh (i3d_texture.cuh), compiled in i3d_texture.cu, a device module of its own: its
 * state, the atlas layout and the call the engine (i3d_engine.cu) makes after it has validated the call and computed the poses.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/i3d_types.h"
#include "i3d_host.h"
#include "i3d_observe.cuh"

namespace i3d
{

// The atlas of F faces at S texels per cell side (texture::layout)
struct TexLayout { int S, cols, rows, W, H; };

// The resident mesh as the bake reads it
struct TexMesh { int32_t F; const float* vpos; const uint8_t* vcol; const int3* faces; };

// The texture of the resident mesh: the atlas [H][W][3] and the UVs [F][3][2] of the last bake, the world -> camera poses [F][12] it
// used (written by the engine), the device counters of k_tex_bake and the event pair of its device time and of the decomposition's
// device time.  The texture's decomposition (texture::decompose) lives here too: the bake's per-texel observation flags, the albedo and
// shading atlases and their counters; it is valid while `intrinsic` and `have` both hold, so whatever drops the texture drops it.
struct TextureState
{
    Dev<uint8_t> rgb; Dev<float> uv; Dev<float> rt; Dev<unsigned long long> counts;
    cudaEvent_t ev[2] = {};
    bool ev_ready = false;
    bool have = false;                  // a texture of the current resident mesh
    int32_t W = 0, H = 0, S = 0, cols = 0; int64_t F = 0;    // atlas size, layout and face count of the texture
    Dev<uint8_t> observed;              // [H][W]: 1 = the bake coloured the texel from the keyframes (k_tex_observed)
    Dev<float> albedo, shading;         // [H][W][3], [H][W] of the last decomposition
    Dev<unsigned long long> dcounts; Dev<unsigned> drange;
    bool intrinsic = false;             // a decomposition of the texture
};

namespace texture
{
// The atlas layout of F > 0 faces at S texels per cell side; false when a side exceeds I3D_TEXTURE_MAX_SIDE
bool layout(int64_t F, int S, TexLayout& L);
// Bakes the texture of mesh m (F > 0 faces) with layout L from the frames fr, the colour frames bgr [F][H][W][3] and the poses in ts.rt
// (the caller validated every argument and wrote ts.rt); the result becomes ts's texture.  info (may be nullptr) gets the counts and
// device time; the observation flags of the decomposition (k_tex_observed) are timed apart as phase "texture_observed".
void bake(TextureState& ts, Timing& tm, const TexMesh& m, const TexLayout& L, const FrameView& fr, const uint8_t* bgr, const SelectCam& cam,
          const CullView& cull, int K, I3DTextureInfo* info, cudaStream_t st);
// Decomposes the texture of ts (the caller checked that it exists and belongs to mesh m, and validated the lighting and min_shading)
// into albedo and shading under `light`; the result becomes ts's decomposition.  info (may be nullptr) gets the counts, the albedo
// range and the device time.
void decompose(TextureState& ts, const TexMesh& m, const ShLight& light, float min_shading, I3DIntrinsicTextureInfo* info, cudaStream_t st);
} // namespace texture

} // namespace i3d
