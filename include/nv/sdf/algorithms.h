// nv/sdf/algorithms.h — the two SDFAlgorithms entry points of the refinement loop's grid-level transitions, with the
// reference's signatures (libintrinsic3d/include/nv/sdf/algorithms.h; src/sdf/algorithms.cpp:200-235, 368-458), computed by
// the H100 engine (i3d_clear_voxels_outside_thin_shell / i3d_upsample_grid) instead of host hash-map passes:
//
//   SDFAlgorithms::clearVoxelsOutsideThinShell(grid, thres_shell);     // Intrinsic3D::prepareGridLevel  (intrinsic3d.cpp:307-313)
//   SparseVoxelGrid<VoxelSBR>* up = SDFAlgorithms::upsample(grid);      // Intrinsic3D::finishGridLevel   (intrinsic3d.cpp:320-331)
//
// Iteration order of the results: survivors keep their relative order; the 8 children of voxel i follow each other in the
// reference's (z, y, x) loop order.  (The reference's own orders are those of std::unordered_map.)
#pragma once
#include <vector>

#include <nv/mat.h>
#include <nv/sparse_voxel_grid.h>

namespace nv
{
namespace SDFAlgorithms
{
// +x,-x,+y,-y,+z,-z (src/sdf/algorithms.cpp:75-91)
std::vector<Vec3i> collectRingNeighborhood(const Vec3i& v_pos);
void clearVoxelsOutsideThinShell(SparseVoxelGrid<VoxelSBR>* grid, double thres_shell);
SparseVoxelGrid<VoxelSBR>* upsample(const SparseVoxelGrid<VoxelSBR>* grid);
// Voxel -> VoxelSBR (sdf_refined = sdf, albedo = 0.6), invalid voxels (weight <= 0) dropped (src/sdf/algorithms.cpp:47-72); host code
SparseVoxelGrid<VoxelSBR>* convert(SparseVoxelGrid<Voxel>* grid);
// CUDA device used by the two functions above (default 0)
void setDevice(int cuda_device);
} // namespace SDFAlgorithms
} // namespace nv
