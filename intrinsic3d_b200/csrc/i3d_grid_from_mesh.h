/*
 * i3d_grid_from_mesh.h — the voxel grid from a triangle mesh (i3d_grid_from_mesh.cuh), compiled in i3d_grid_from_mesh.cu, a device module
 * of its own: its scratch, the per-voxel results of the last conversion, and the calls the engine (i3d_engine.cu) makes after it has
 * validated them.  The engine compacts the kept candidates and installs the voxel set.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>

#include "../../include/i3d_types.h"
#include "i3d_distance.h"
#include "i3d_host.h"

namespace i3d
{

struct GridFromMeshState
{
    DistGridScratch grid;                               // the search grid of the source mesh
    // welding: vertex sort keys and order, and per vertex its weld representative (the lowest index at its position)
    Dev<uint32_t> wk32, wk32b; Dev<unsigned long long> wk64, wk64b; Dev<int32_t> wi, wi2, weld;
    // incidences 3 f + k: welded-vertex and welded-edge keys and their sorted order; per face its unit normal, per corner the vertex
    // pseudonormal, per edge slot k (corners k, k + 1) the edge pseudonormal and the boundary flag; per welded vertex the boundary flag
    Dev<uint32_t> vk, vk2; Dev<unsigned long long> ek, ek2; Dev<int32_t> vi, vi2, ei, ei2;
    Dev<double> fn, vn, en; Dev<uint8_t> eb, vb;
    // candidate bricks (sorted, unique key) and the per-candidate query results
    Dev<unsigned long long> bk, bk2; Dev<int64_t> nsel;
    Dev<uint8_t> keep; Dev<double> sdf; Dev<int32_t> face; Dev<int8_t> feat;
    Dev<unsigned long long> counters;
    Dev<uint8_t> cub;
    int64_t num_bricks = 0;
    // the last successful conversion: per voxel the nearest face and feature
    Dev<int32_t> last_face; Dev<int8_t> last_feat; int64_t last_n = 0;
    bool have_last = false;
    cudaEvent_t ev[8] = {};
    bool ev_ready = false;
};

namespace gfm
{
// Runs everything up to the keep flags for mesh m (F > 0) with parameters the caller validated: the candidate bricks, welding and
// pseudonormals, the search grid and the per-voxel query.  Fills *info but its install time.  Returns non-zero with the message in
// `error`, having written no engine state, when a cap or the coordinate range is exceeded.  On success s.keep [info->num_candidate_voxels] holds bit 1 for each emitted voxel.
int query(GridFromMeshState& s, const DistMesh& m, const I3DGridFromMeshParams& p, I3DGridFromMeshInfo& info, std::string& error, cudaStream_t st);
// Writes the m kept candidates act[0..m) into the voxel arrays, and their face and feature into s.last_*
void gather(GridFromMeshState& s, const int32_t* act, int64_t m, const VoxelArrays& out, cudaStream_t st);
} // namespace gfm

} // namespace i3d
