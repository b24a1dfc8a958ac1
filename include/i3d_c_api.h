/*
 * i3d_c_api.h — C-ABI of the H100-native joint-refinement engine (libi3d_b200.so).
 *
 * This is the drop-in boundary for the ONE hot path of NVlabs/intrinsic3d that this
 * repository replaces: Optimizer::optimize's outer Gauss-Newton iteration
 * (libintrinsic3d/src/refinement/optimizer.cpp:109-173) including everything it does
 * through NLSSolver (src/refinement/nls_solver.cpp:172-394) and Ceres.  The reference has
 * no FFI of its own (everything is statically linked C++); the host shims in
 * include/nv/refinement/ (Optimizer, NLSSolver, cost-term create()) are what bind to
 * these entry points — see INTEGRATION.md.
 *
 * Conventions: plain pointers and sizes only; every array is caller-owned HOST memory and is
 * copied during the call (pinned memory makes the copies asynchronous-capable but is not
 * required); one handle is not thread-safe; every function returns 0 on success, non-zero
 * on error with a message available from i3d_last_error().  There is NO CPU fallback:
 * i3d_engine_create fails if no sm_90 (H100) device is present.
 *
 * Each entry point cites the reference interface it replaces (paths relative to
 * libintrinsic3d/).
 */
#ifndef I3D_C_API_H_
#define I3D_C_API_H_

#include <stdint.h>
#include "i3d_types.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct I3DEngine I3DEngine;

/* Library/ABI version and struct sizes (checked by the host bindings). */
int         i3d_abi_version(void);
uint64_t    i3d_sizeof_params(void);
uint64_t    i3d_sizeof_iter_info(void);

/* Fills *p with data/intrinsic3d.yml defaults (first outer iteration) and the Ceres 2.1.0
 * solver defaults the reference inherits (src/refinement/nls_solver.cpp:300-337). */
void        i3d_default_params(I3DParams* p);

/* Creates an engine on CUDA device `device`.  Replaces: construction of Optimizer +
 * NLSSolver + ceres::Problem (include/nv/refinement/optimizer.h:118, nls_solver.cpp:105-141). */
int         i3d_engine_create(int device, I3DEngine** out);
void        i3d_engine_destroy(I3DEngine* e);
const char* i3d_last_error(const I3DEngine* e);   /* e may be NULL: last create() error */

/* Flattened SparseVoxelGrid<VoxelSBR> (include/nv/sparse_voxel_grid.h:69-161), one entry per
 * hash node IN THE HOST'S ITERATION ORDER (voxel_idx of optimizer.cpp:148-149):
 *   xyz[3n] voxel coordinates, sdf0 = VoxelSBR::sdf, sdf_refined, albedo, weight, rgb[3n] = color.
 * voxel_size = SparseVoxelGrid::voxelSize() (float); truncation = 5*voxel_size (sparse_voxel_grid.cpp:48).
 * Builds the device neighbour table (the engine's replacement for unordered_map::find). */
int         i3d_upload_grid(I3DEngine* e, int64_t n, const int32_t* xyz, const double* sdf0,
                            const double* sdf_refined, const double* albedo, const float* weight,
                            const uint8_t* rgb, float voxel_size);

/* Only the mutable voxel parameters (what Ceres writes through the double* of
 * shading_cost.cpp:89-118): cheaper than re-uploading the grid between optimize() calls. */
int         i3d_upload_voxel_params(I3DEngine* e, const double* sdf_refined, const double* albedo);

/* Per-keyframe images at the pyramid level being optimised: lum = Pyramid::intensity(lvl)
 * (float luminance in [0,1]), depth = Pyramid::depth(lvl) (metres), both [F][H][W] contiguous;
 * pyr_scale = 2^-lvl (ShadingCostData, include/nv/refinement/shading_cost.h:52-73;
 * optimizer.cpp:124-127). */
int         i3d_upload_frames(I3DEngine* e, int32_t F, int32_t W, int32_t H, const float* lum,
                              const float* depth, double pyr_scale);

/* Optimizer::ImageFormationModel (include/nv/refinement/optimizer.h:107-115): poses[6F]
 * world->camera (angle-axis, translation), intrinsics[4] = fx,fy,cx,cy at full resolution,
 * distortion[5] = k1,k2,k3,p1,p2. */
int         i3d_set_camera(I3DEngine* e, const double* poses, const double* intrinsics,
                           const double* distortion);

/* Optimizer::Data::voxel_sh_coeffs (optimizer.h:97): 9 doubles per voxel, same order as the
 * grid arrays; rows of voxels outside the thin shell are never read (Q22). */
int         i3d_set_sh(I3DEngine* e, const double* sh9n);

/* ONE outer iteration of Optimizer::optimize (optimizer.cpp:119-171): observation selection,
 * residual collection, weight normalisation, parameter fixing, LM solve that stops at the
 * first successful step.  State (sdf_refined, albedo, poses, intrinsics, distortion) is
 * updated on the device.  info mirrors NLSSolver::ProblemInfo/SolverInfo.
 * Frame-count limit: k_eg_accum holds the camera sums of all F frames plus K x 8 KB of parked rows in one block's shared memory,
 * (33F + 43) * 8 + K * 8 KB bytes next to its static buffers, against the device's opt-in limit per block (227 KB on H100): about
 * 629 frames at K = 8 (measured on H100) or about 720 at K = 5.  Beyond it the call fails before launching anything, with a message that names F, K and the
 * largest F allowed; the engine stays usable (fewer frames or a smaller K). */
int         i3d_gn_iteration(I3DEngine* e, const I3DParams* params, I3DIterInfo* info);

/* Reads the refined parameters back (the in-place mutation the reference performs through
 * raw pointers).  Any pointer may be NULL. */
int         i3d_download_state(I3DEngine* e, double* sdf_refined, double* albedo, double* poses,
                               double* intrinsics, double* distortion);

/* ---- SVSH lighting: the producer of voxel_sh_coeffs (SURVEY.md §8 a15 / f1) ---- */
uint64_t    i3d_sizeof_lighting_params(void);
uint64_t    i3d_sizeof_lighting_info(void);
/* Intrinsic3D::Config defaults (include/nv/refinement/intrinsic3d.h:81-82) + Ceres 2.1.0 defaults. */
void        i3d_default_lighting_params(I3DLightingParams* p);

/* LightingSVSH::estimate() followed by LightingSVSH::computeVoxelShCoeffs()
 * (src/lighting/lighting_svsh.cpp:166-346 and :93-110; called back to back by Intrinsic3D::refine,
 * src/refinement/intrinsic3d.cpp:255-268) on the grid currently on the device (uses sdf_refined,
 * albedo, weight, rgb): Subvolumes::compute (src/lighting/subvolumes.cpp:66-96,211-239), one data
 * row per in-shell voxel, 9 smoothness rows per directed pair of neighbouring subvolumes, Ceres
 * trust-region LM + CGNR + block-Jacobi up to max_iterations; then the per-voxel trilinear blend
 * of the 8 surrounding subvolume vectors.  The per-voxel result REPLACES what i3d_set_sh uploaded
 * (it is the `sh` input of the following i3d_gn_iteration calls).  Returns 0 on success;
 * info->usable == 0 reproduces estimate() returning false.  Subvolumes are numbered in ascending
 * (z, y, x) order of their integer index (the reference's order is that of a std::unordered_map,
 * i.e. unspecified; nothing downstream depends on it). */
int         i3d_estimate_lighting(I3DEngine* e, const I3DLightingParams* params, I3DLightingInfo* info);
/* Subvolumes::count() of the last estimate. */
int64_t     i3d_lighting_num_subvolumes(const I3DEngine* e);
/* Subvolumes::index(i) (3 ints each) and LightingSVSH::shCoeffs() (9 doubles each).  Either may be NULL. */
int         i3d_download_lighting(I3DEngine* e, int32_t* subvolume_index3, double* sh9);
/* Optimizer::Data::voxel_sh_coeffs as i3d_estimate_lighting left it (or i3d_set_sh uploaded it):
 * sh9n[9*i..] per voxel; has_sh[i] = 0 where the reference leaves an empty vector (invalid voxel or
 * outside the thin shell; zeros are written there).  has_sh may be NULL. */
int         i3d_download_voxel_sh(I3DEngine* e, double* sh9n, uint8_t* has_sh);

/* ---- voxel recolouring: the step right after the path (SURVEY.md §8 f2) ---- */
/* Pyramid::color(lvl) of every frame (include/nv/rgbd/pyramid.h): F*H*W*3 bytes, interleaved B,G,R like the reference's
 * cv::Mat (CV_8UC3); same F, W, H as the last i3d_upload_frames (call that first). */
int         i3d_upload_color_frames(I3DEngine* e, const uint8_t* bgr);
/* Intrinsic3D::recomputeColors (src/refinement/intrinsic3d.cpp:381-409) = SDFColorization::add for every frame +
 * SDFColorization::compute (src/sdf/colorization.cpp:113-189): for every voxel with a forward-difference normal, the
 * observations (weight > 0) over all frames at the current intrinsics / distortion, the best max_num_observations of
 * them (0 = all), weighted mean of their bilinearly fetched colours; voxels without an observation keep their colour.
 * pose_world_to_cam: the Mat4f the reference passes to add() for every frame, as [F][12] floats (rotation row-major 9,
 * translation 3); NULL = math::poseVecAAToMat(current pose).cast<float>() like recomputeColors does.
 * Updates the device copy of the voxel colours (E_a weights and the lighting estimate read it).  Outputs may be NULL. */
int         i3d_recompute_colors(I3DEngine* e, const float* pose_world_to_cam, float max_occlusion_distance,
                                 int32_t max_num_observations, int64_t* num_recolored, int64_t* num_observations);
/* VoxelSBR::color of every voxel (3 bytes r,g,b each) as the device holds it. */
int         i3d_download_colors(I3DEngine* e, uint8_t* rgb3n);

/* ---- grid-level transitions: the voxel set changes on the device (SURVEY.md §8 f3) ---- */
/* SparseVoxelGrid::numVoxels() of the grid currently on the device. */
int64_t     i3d_num_voxels(const I3DEngine* e);
/* SDFAlgorithms::clearVoxelsOutsideThinShell(grid, thres_shell) (src/sdf/algorithms.cpp:368-458; called by
 * Intrinsic3D::prepareGridLevel, src/refinement/intrinsic3d.cpp:307-313): keeps every valid voxel with
 * |sdf_refined| <= thres_shell plus its existing +-x,+-y,+-z,+2x,+2y,+2z neighbours, and every other voxel that has a
 * voxel of the opposite sign within its 5x5x5 neighbourhood; removes the rest.  Survivors keep their relative order (the
 * reference's order after unordered_map::erase is unspecified).  Per-voxel SH and the shard are invalidated. */
int         i3d_clear_voxels_outside_thin_shell(I3DEngine* e, double thres_shell, int64_t* num_voxels_out);
/* SDFAlgorithms::upsample<VoxelSBR>(grid) (src/sdf/algorithms.cpp:200-235 with interpolate<VoxelSBR> :118-197; called by
 * Intrinsic3D::finishGridLevel, intrinsic3d.cpp:320-331): voxel size halves, every voxel i becomes 8 voxels
 * 2p + (x,y,z) stored at 8i + (4z + 2y + x), each the float trilinear blend at p + (x,y,z)/2 of the valid corners of p's
 * unit cube (weight 0 when at most 4 of the 8 corners are valid). */
int         i3d_upsample_grid(I3DEngine* e, int64_t* num_voxels_out);
/* The grid as the device holds it (after pruning / upsampling the host needs the new coordinates): xyz[3n], sdf0[n]
 * (VoxelSBR::sdf), sdf_refined[n], albedo[n], weight[n], rgb[3n], voxel size.  Any pointer may be NULL. */
int         i3d_download_grid(I3DEngine* e, int32_t* xyz, double* sdf0, double* sdf_refined, double* albedo,
                              float* weight, uint8_t* rgb, float* voxel_size);

/* ---- multi-GPU (one process per GPU; voxel ranges sharded, see DESIGN.md §multi-GPU) ---- */
/* 128-byte NCCL unique id created on rank 0 and distributed by the host (e.g. torch.distributed). */
int         i3d_comm_unique_id(uint8_t id128[128]);
int         i3d_comm_init(I3DEngine* e, int32_t rank, int32_t world, const uint8_t id128[128]);
/* Peer-memory exchange (optional, after i3d_comm_init): the packed partial sums of the PCG loop are exchanged by pulling the peers'
 * buffers over NVLink from inside the engine's own kernels instead of ncclAllReduce.  export: allocates this rank's mailbox and returns
 * its 64-byte CUDA IPC handle; the host gathers the handles of all ranks (rank order) and passes them to connect on every rank.
 * Without these two calls the engine uses ncclAllReduce.  (No reference counterpart: the reference is single-process.) */
int         i3d_comm_p2p_export(I3DEngine* e, uint8_t handle64[64]);
int         i3d_comm_p2p_connect(I3DEngine* e, const uint8_t* handles /* [world][64] */);

/* Rows (voxels) this rank owns: [begin, end) in the grid's iteration order. */
int         i3d_set_shard(I3DEngine* e, int64_t voxel_begin, int64_t voxel_end);

/* ---- measurement / parity hooks (used by tests and bench.py; not needed by a drop-in) ---- */
/* Device time (ms) of the named phase during the last i3d_gn_iteration, from CUDA events on the
 * engine's stream; also launch counts.  Names: "select", "build", "scale", "pcg", "candidate",
 * "total"; per-kernel: "k_eg_apply" (sum over launches) with count via i3d_phase_count. */
double      i3d_phase_ms(const I3DEngine* e, const char* name);
/* level 0 (default): phase events and every launch of k_eg_rows (Jacobian build / cost), k_eg_apply and k_select_obs are timed;
 * level 1: every kernel of the iteration (an event between two kernels suppresses their programmatic-dependent-launch
 * overlap, so the per-kernel table is taken on a separate, untimed step). */
int         i3d_debug_set_kernel_timers(I3DEngine* e, int level);
int64_t     i3d_phase_count(const I3DEngine* e, const char* name);
/* E_g row slots of the last iteration: slot s = k*num_active + a.  Any pointer may be NULL.
 * voxel[s], frame[s] (-1 = empty slot), residual[s] (unweighted), raw_weight[s] (0 = invalid row),
 * jac[29*S] column-major raw (unweighted, unscaled) Jacobian — only when keep_raw_jacobian was set. */
int64_t     i3d_debug_num_slots(const I3DEngine* e);
int         i3d_debug_set_keep_raw_jacobian(I3DEngine* e, int keep);
int         i3d_debug_get_rows(I3DEngine* e, int32_t* voxel, int32_t* frame, double* residual,
                               double* raw_weight, float* jac_colmajor);
/* observation selection of the last iteration for ALL voxels: frames[n*K] (-1 none), weights[n*K],
 * active[n]; layout [n][K], descending priority. */
int         i3d_debug_get_observations(I3DEngine* e, int32_t K, int32_t* frames, float* weights,
                                       uint8_t* active);
/* last evaluated LM trial step in unknown space [sdf n | albedo n | poses 6F | intr 4 | dist 5]
 * (unscaled delta), the free mask and the Jacobi column scale. */
int         i3d_debug_get_step(I3DEngine* e, double* step, uint8_t* free_mask, double* col_scale);
/* normal-equation pieces of the last iteration (build_only = 1 is enough), unknown space [U = 2n + 6F + 9]: b[U] = J'^T f (Jacobi
 * scaled gradient), s[U] (Jacobi column scale, 0 for fixed unknowns), jtj[U] = s^2 * column norm^2, and the raw (unweighted by the
 * type weight, unscaled) E_g camera sums cam_acc[33F + 43]: per frame 6 gradient (sum w_raw r J), 6 column norms, the upper 6x6
 * triangle row by row (21); then 9 gradient, 9 column norms of intrinsics | distortion, the upper 4x4 (10) and 5x5 (15) triangles.
 * Any pointer may be NULL. */
int         i3d_debug_get_normal_equations(I3DEngine* e, float* b, float* s, float* jtj, float* cam_acc);
/* q[U] = S (J^T W J) S v for the rows of the last iteration (all four terms, no D^2 term): the raw operator output of the production
 * k_eg_apply + k_op_partial pair times s, in float.  Leaves nothing behind that a following i3d_gn_iteration reads.  Single GPU only. */
int         i3d_debug_apply_operator(I3DEngine* e, const float* v, float* q);

#ifdef __cplusplus
}
#endif
#endif /* I3D_C_API_H_ */
