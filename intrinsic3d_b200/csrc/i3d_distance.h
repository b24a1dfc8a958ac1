/*
 * i3d_distance.h — the distance between the resident mesh and a reference mesh (i3d_distance.cuh), compiled in i3d_distance.cu, a device
 * module of its own: its state (the reference mesh, the search-grid scratch and the last results) and the calls the engine
 * (i3d_engine.cu) makes after it has validated them.
 */
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/i3d_c_api.h"
#include "../../include/i3d_types.h"
#include "i3d_host.h"
#include "i3d_track.h"

namespace i3d
{

// A triangle mesh as the distance kernels read it
struct DistMesh { int64_t V, F; const float* vpos; const int3* faces; };

// The search grid of a target mesh (i3d_distance.cuh); off / cnt / faces are null while it is being counted
struct DistGrid
{
    float lo[3]; float h; int n[3];
    double margin;
    const int64_t* off; const int32_t* cnt; const int32_t* faces;
};

// What sizing and filling one search grid needs: per cell its face count and the int64 offset of its run in cell_faces, the bounds
// partials and the entry counter
struct DistGridScratch
{
    Dev<int32_t> cell_count, cell_faces; Dev<int64_t> cell_off; Dev<uint8_t> cub;
    Dev<double> partials;
    Dev<unsigned long long> counter;
};

// Reference mesh, grid scratch and results of the distance calls of one engine
struct DistanceState
{
    Dev<float> ref_vpos; Dev<int3> ref_faces;
    int64_t ref_V = 0, ref_F = 0;
    bool have_ref = false;
    DistGridScratch grid;                  // search grid of the current target
    Dev<double> partials, stats;           // per-block partials and the finished statistics of both directions
    Dev<unsigned long long> vtests;
    // the last results: per-vertex distance and face of the resident mesh, and (when keep) the per-sample (d^2, face) of both directions
    Dev<float> vdist; Dev<int32_t> vface; int64_t result_V = 0;
    bool have_result = false;
    bool keep = false;
    Dev<float> keep_d2[2]; Dev<int32_t> keep_face[2]; int64_t keep_n[2] = {0, 0};
    bool have_keep = false;
    cudaEvent_t ev[14] = {};
    bool ev_ready = false;
    // the reference-mesh registration (i3d_register.cuh), which builds its grid in `grid`: the pose state, the block partials, every
    // system of the last call with the pose M it was formed at, the first system's per-sample faces and sum w of the first and last system
    Dev<TrackState> reg_state; Dev<double> reg_T, reg_partials, reg_wpartials, reg_sums, reg_sys, reg_poses; Dev<int32_t> reg_face;
    Dev<unsigned long long> reg_counters;
    int reg_n = 0; int64_t reg_samples = 0; double reg_wsum[2] = {0.0, 0.0};
    bool have_reg = false;
    std::vector<cudaEvent_t> reg_ev;
};

namespace distance
{
// The search grid of target t (F > 0) for queries within max_distance: its size, cell edge (cell_size, or twice the mean edge length
// when 0), margin and entry count, and when bounds is set the faces' AABB (min x, y, z, max x, y, z).  Returns false with the message
// when a cap is exceeded.
bool plan(DistGridScratch& s, const DistMesh& t, float cell_size, float max_distance, DistGrid& g, int64_t& entries, double* bounds, std::string& error,
          cudaStream_t st);
// Counts, scans and fills the planned grid g of target t into s, and points g at it
void build(DistGridScratch& s, const DistMesh& t, DistGrid& g, int64_t entries, cudaStream_t st);
// Uploads the reference mesh after checking it on the host; returns non-zero with the message in `error`, keeping the previous one
int upload_reference(DistanceState& ds, int64_t V, const float* xyz, int64_t F, const int32_t* faces, std::string& error, cudaStream_t st);
// Both directions and the vertex query between the resident mesh a (F > 0) and the reference (present), with parameters the caller
// validated.  Returns non-zero with the message in `error`, writing nothing, when a search grid exceeds its cell or entry cap.
int compute(DistanceState& ds, const DistMesh& a, const I3DDistanceParams& p, I3DDistanceInfo* info, std::string& error, cudaStream_t st);
// False with the message when T [12] (R row-major | t) is not finite or R is not a rotation: max |R^T R - I| > 1e-5 or det R < 0
bool check_rigid(const double* T, std::string& error);
// Registers the reference (present) to the resident mesh a (F > 0) from T_init (nullptr: identity; checked by the caller, as are the
// parameters) into T_out [12] (DESIGN.md §6aa).  Returns non-zero with the message in `error`, writing nothing, when the search grid
// exceeds its cell or entry cap.
int register_reference(DistanceState& ds, const DistMesh& a, const I3DRegisterParams& p, const double* T_init, double* T_out, I3DRegisterInfo* info,
                       std::string& error, cudaStream_t st);
// Moves the reference (present) by T (checked by the caller) on the device
void transform_reference(DistanceState& ds, const double* T, cudaStream_t st);
} // namespace distance

} // namespace i3d
