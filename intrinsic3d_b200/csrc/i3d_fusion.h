/*
 * i3d_fusion.h — the RGB-D fusion (i3d_fusion.cuh, DESIGN.md §6h), compiled in i3d_fusion.cu, a device module of its own: the state of a
 * fusion in progress, and the calls the engine (i3d_engine.cu) makes with its stream.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>

#include "../../include/i3d_types.h"
#include "i3d_fusion_view.cuh"
#include "i3d_grid.cuh"
#include "i3d_host.h"

namespace i3d
{

// RGB-D fusion in progress: its own hash table and Voxel arrays, one entry per hash slot, and scratch that only grows
struct FusionState
{
    bool active = false;
    I3DFusionParams p{};
    uint64_t cap = 0;                  // hash slots (a power of two)
    int64_t n = 0;                     // allocated voxels
    Dev<unsigned long long> keys; Dev<unsigned> vals;
    Dev<int32_t> x, y, z; Dev<float> sdf, w, sdf2, w2; Dev<uchar4> rgb;
    Dev<int> ctl;                      // [0] allocated voxels, [1] alloc status, [2] correctSDF "changed", [3] valid voxels
    Dev<float> depth_in, depth, nrm; Dev<uint8_t> bgr;      // host frames of i3d_fusion_integrate; the eroded depth and its normals
    Dev<unsigned long long> sk, sk2; Dev<int32_t> si, si2; Dev<uint8_t> cub;
    // the odometry's motion state (track::odometry): the last `motion` (0..2) integrated camera -> world poses, R row-major | t in
    // double, newest in motion_T[1]; begin and every integrate clear it
    int motion = 0;
    double motion_T[2][12] = {};
    // the reference of the _ref odometry (DESIGN.md §6q): the last frame the loop integrated (-1: none) and its camera -> world pose;
    // kept and cleared with the motion state, and cleared by i3d_sensor_frames_begin, since it indexes the sensor store
    int32_t ref_id = -1;
    double ref_T[12] = {};
};

namespace fusion
{
// Starts a fusion with P (validated by the caller): an empty table of the initial capacity.  The fusion phases start from zero and add
// up over the calls until the finish.
void begin(FusionState& fs, Timing& tm, const I3DFusionParams& P, cudaStream_t st);
// Uploads F host frames (depth [F][dc], colour [F][cc][3]) into fs's upload scratch and integrates them with integrate()
int integrate_host(FusionState& fs, Timing& tm, int F, const I3DFusionCamera& dc, const float* depth, const I3DFusionCamera& cc, const uint8_t* bgr,
                   const float* pose_cam_to_world, const float* pose_world_to_cam, std::string& error, cudaStream_t st);
// The loop body of AppFusion::fuseSDF for n frames already on the device: frame f is depth[ids[f]] / bgr[ids[f]] (frame f when ids is
// nullptr), with pose row f.  Erosion writes into fs.depth, so the source planes are only read.  Returns non-zero with the message in
// `error` when a frame allocates voxels outside the device hash's range or the table would exceed 2^30 voxels.
int integrate(FusionState& fs, Timing& tm, int n, const I3DFusionCamera& dc, const float* depth, const I3DFusionCamera& cc, const uint8_t* bgr,
              const int32_t* ids, const float* pose_cam_to_world, const float* pose_world_to_cam, std::string& error, cudaStream_t st);
// The correctSDF sweeps (timed as "fusion_correct", counted in "fusion_sweeps"); nothing without allocated voxels
void correct(FusionState& fs, Timing& tm, cudaStream_t st);
// Sorts the volume into canonical order: fs.si[0..) = volume indices.  valid_only: voxels with weight <= 0 sort last and are not counted.
// Returns the number of voxels in the order (valid ones only when valid_only); 0 without allocated voxels.
int sort(FusionState& fs, bool valid_only, cudaStream_t st);
// SDFAlgorithms::convert of the first m voxels of the order into out
void convert(const FusionState& fs, int m, const VoxelArrays& out, cudaStream_t st);
// The volume in progress, read-only, for a reader outside this module (i3d_fusion_view.cuh)
FuseView view(const FusionState& fs);
// The volume in canonical order, interleaved, into host buffers (each may be nullptr)
void download(FusionState& fs, int32_t* xyz, float* sdf, float* weight, uint8_t* rgb, cudaStream_t st);
} // namespace fusion

} // namespace i3d
