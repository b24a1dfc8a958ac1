/*
 * i3d_mesh.h — the surface extraction (i3d_mesh.cuh) and its colour modes (i3d_vis.cuh), compiled in i3d_mesh.cu, a device module of
 * its own: its state, and the two calls the engine (i3d_engine.cu) makes with the grid it builds and its stream.
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

struct MeshGrid
{
    int64_t n;
    const int32_t* x; const int32_t* y; const int32_t* z;
    const double* sdf;              // sdf0 or the refined sdf
    const float* weight;
    const uchar4* rgb;
    const int32_t* nbr;             // [12][n]
    const unsigned long long* keys; const int32_t* vals; uint64_t mask;    // device hash of the grid, for the (1,1,1) corner
    float voxel_size;
};

// Corner buffers of the raw triangle soup, corner index = 3 * face + k: position, colour and the position's sort key (float bits
// with the sign of zero canonicalised: -0.0 and +0.0 compare equal, as in merge's std::map).
struct MeshCorners
{
    float* pos;                    // [3M]
    uint8_t* col;                  // [3M]
    uint32_t* key_lo;              // z bits
    unsigned long long* key_hi;    // x bits << 32 | y bits
};

// Surface-extraction state of an engine: scratch that only grows, the event pairs of the stage timings, the resident mesh of the last
// extraction (pointers into the scratch) and the per-voxel colours of the last colour pass
struct MeshState
{
    Dev<uint8_t> cases, keep, cub; Dev<int32_t> cnt, sel; Dev<int64_t> off; Dev<unsigned long long> cubes, best;
    Dev<float> cpos, vpos, vpos2; Dev<uint8_t> ccol, vcol, vcol2;
    Dev<uint32_t> klo, klo2; Dev<unsigned long long> khi, khi2;
    Dev<int32_t> perm, perm2, first, fid, head, seg, cvid, parent, used, newid;
    Dev<int3> faces, faces2; Dev<unsigned> ccount, cminf;
    cudaEvent_t ev[16] = {};           // begin / end of up to 8 device-only segments of one extraction
    bool ev_ready = false;
    bool have_mesh = false;
    int64_t mesh_V = 0, mesh_F = 0;
    float* mesh_vpos = nullptr; uint8_t* mesh_vcol = nullptr; int3* mesh_faces = nullptr;
    Dev<uchar4> vis_rgb;
    // simplification (mesh::simplify): per vertex its cluster, per cluster its sorted runs of vertices and corners, the corners sorted
    // by cluster, per face its quadric [9][F] and its cluster ids, the cluster representatives, and two output slots, so that the result
    // never overwrites the resident mesh it is computed from.  The cell and face sorts use the welding's sort scratch above.
    Dev<int32_t> s_bad, s_cid, s_run, s_corner, s_corner2, s_cstart, s_cend; Dev<uint32_t> s_ckey, s_ckey2;
    Dev<double> s_quad; Dev<int3> s_cfaces; Dev<float> s_rpos; Dev<uint8_t> s_rcol; Dev<unsigned long long> s_counts;
    Dev<float> s_vpos[2]; Dev<uint8_t> s_vcol[2]; Dev<int3> s_faces[2];
};

namespace mesh
{
// The colour pass (i3d_vis.cuh) of mode 1 .. I3D_MESH_COLOR_COUNT - 1 (validated by the caller) into ms.vis_rgb [g.n], timed as phase
// "mesh_colorize".  g.sdf is the sdf the mesh is cut from, sg / sub_sh [S][9] the subvolumes and subvolume SH of the last lighting
// estimate (read by the shading modes only).  Writes nothing but ms.vis_rgb.
void colorize(MeshState& ms, Timing& tm, const GridView& g, const SubvolGrid& sg, const double* sub_sh, int S, int mode, cudaStream_t st);
// Marching cubes over g, welding, degenerate-face removal and (optionally) the largest component, into the resident mesh of ms.  Every
// count is read back before the buffers of the next stage are sized; info (may be nullptr) gets the counts and stage times.  Returns
// non-zero with the message in `error`, writing no info and leaving no mesh resident, when the triangles exceed the int32 corner indices.
int extract(MeshState& ms, const MeshGrid& g, bool largest_component_only, I3DMeshInfo* info, std::string& error, cudaStream_t st);
// Quadric-error vertex clustering of the resident mesh of ms (which the caller checked exists) with cells of edge cell_size (finite,
// > 0, checked by the caller); the result becomes the resident mesh.  info (may be nullptr) gets the counts and stage times.  Returns
// non-zero with the message in `error`, leaving the resident mesh as it was and writing no info, when a cell coordinate is not finite
// or outside int32.
int simplify(MeshState& ms, float cell_size, I3DSimplifyInfo* info, std::string& error, cudaStream_t st);
} // namespace mesh

} // namespace i3d
