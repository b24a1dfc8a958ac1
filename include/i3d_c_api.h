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

/* ---- RGB-D fusion: the producer of the grid (DESIGN.md §6h) ---- */
uint64_t    i3d_sizeof_fusion_params(void);
/* voxel_size 0.004, depth range [0.1, 4.0], integration_weight_sample 10, no clipping, discont_window_size 2,
 * correct_sdf_iterations 10, default capacity. */
void        i3d_default_fusion_params(I3DFusionParams* p);
/* Starts an empty fusion volume (SparseVoxelGrid<Voxel>::create + setClipBounds, app_fusion.cpp:123-139).  The grid the engine
 * currently holds is left alone until i3d_fusion_finish.  Fails for voxel_size <= 1e-5 (as create() returns nullptr) and on an
 * engine with world > 1 (fusion runs on one GPU). */
int         i3d_fusion_begin(I3DEngine* e, const I3DFusionParams* params);
/* Fuses F frames in order, each as the loop body of AppFusion::fuseSDF (app_fusion.cpp:146-165): erodeDiscontinuities,
 * computeNormals (only when integration_weight_sample > 0, the only case that reads them), then SparseVoxelGrid::integrate
 * (computeFrustumBounds, alloc, per-voxel update; src/sparse_voxel_grid.cpp:300-395, 572-602).
 *   depth    float metres [F][depth_cam.height][depth_cam.width], already range-thresholded as the sensor classes do
 *   bgr      uint8 [F][color_cam.height][color_cam.width][3], interleaved B,G,R like i3d_upload_color_frames
 *   pose_cam_to_world, pose_world_to_cam   float [F][12]: rotation row-major (9), translation (3)
 * Divergence: integrate() inverts the camera-to-world Mat4f itself with Eigen's 4x4 float inverse (sparse_voxel_grid.cpp:305),
 * which is not restated bit for bit; the caller supplies both directions instead (as i3d_recompute_colors takes pose_world_to_cam).
 * Fails with a message when a voxel to allocate lies outside the +-2^20 coordinate range of the device hash. */
int         i3d_fusion_integrate(I3DEngine* e, int32_t F, const I3DFusionCamera* depth_cam, const float* depth,
                                 const I3DFusionCamera* color_cam, const uint8_t* bgr,
                                 const float* pose_cam_to_world, const float* pose_world_to_cam);
/* After the last frame (app_fusion.cpp:167-173): SDFAlgorithms::correctSDF (src/sdf/algorithms.cpp:260-337, run as Jacobi sweeps:
 * DESIGN.md §6h), clearInvalidVoxels (:342-363), SDFAlgorithms::convert (sdf0 = sdf_refined = sdf, albedo 0.6), then the result
 * becomes the engine's grid exactly as i3d_upload_grid of it would: voxel size, truncation, hash and neighbour tables.  Voxels are
 * in canonical 8^3-brick-major order (sorted by floor(c/8) z,y,x then c mod 8 z,y,x).  Per-voxel SH, the shard and the last
 * iteration are invalidated.  Ends the fusion.  An empty result leaves an empty grid (num_voxels_out = 0). */
int         i3d_fusion_finish(I3DEngine* e, int64_t* num_voxels_out);

/* ---- surface extraction: the grid as a coloured triangle mesh (DESIGN.md §6j) ---- */
uint64_t    i3d_sizeof_mesh_info(void);
/* MarchingCubes<VoxelSBR>::extractMesh + MeshUtil::removeDegenerateFaces (src/mesh/marching_cubes.cpp:64-317, src/mesh/util.cpp:168-198)
 * and, with largest_component_only, removeLooseComponents + removeUnusedVertices (util.cpp:47-165), over the resident grid.  The mesh
 * stays on the device until i3d_download_mesh; *info (may be NULL) gets the counts of every stage and its device time.
 * Faces are in (voxel index, triangle slot) order; vertex ids in order of first appearance over the face corners; two corners are one
 * vertex iff their float positions compare equal; without the component filter, vertices that only degenerate faces used are kept.
 * Reads the grid only: state, camera, lighting, frames and the last iteration are unchanged.  A change of the voxel set (upload,
 * prune, upsample, fusion) drops the resident mesh.  Fails without a grid and for an sdf_source other than 0 or 1. */
int         i3d_extract_mesh(I3DEngine* e, const I3DMeshParams* params, I3DMeshInfo* info);
/* i3d_extract_mesh with the mesh coloured by a colour mode of SDFVisualization::colorize (src/sdf/visualization.cpp:101-164; color_mode:
 * I3D_MESH_COLOR_*).  I3D_MESH_COLOR_VOXEL is i3d_extract_mesh itself; any other mode first computes every voxel's colour in that mode on
 * the device (the geometric modes from the sdf the mesh is cut from) and extracts with those colours.  The shading modes blend the
 * subvolume SH of the last i3d_estimate_lighting.  The mesh replaces the resident mesh that i3d_download_mesh reads; the device time
 * of the colour pass is i3d_phase_ms("mesh_colorize").  The voxel colours and every other engine state are left alone.  Fails, as
 * i3d_extract_mesh does, without a grid or for a bad sdf_source, and for a bad color_mode or a shading mode without a lighting estimate
 * of the current voxel set (the per-voxel SH of i3d_set_sh is not one). */
int         i3d_extract_mesh_colored(I3DEngine* e, const I3DMeshParams* params, int32_t color_mode, I3DMeshInfo* info);
/* The colours of every voxel in a colour mode: rgb uint8 [n][3], in the grid's order; sdf_source as in I3DMeshParams.  Mode
 * I3D_MESH_COLOR_VOXEL gives the voxel colours.  Writes no engine state; fails as i3d_extract_mesh_colored does. */
int         i3d_mode_colors(I3DEngine* e, int32_t sdf_source, int32_t color_mode, uint8_t* rgb);
/* The resident mesh: xyz float [V][3] metres, rgb uint8 [V][3], faces int32 [F][3] (V, F: info->num_vertices / num_faces).  Any
 * pointer may be NULL.  Fails when no mesh of the current grid has been extracted. */
int         i3d_download_mesh(I3DEngine* e, float* xyz, uint8_t* rgb, int32_t* faces);

/* ---- simplifying the resident mesh by quadric-error vertex clustering (DESIGN.md §6s) ---- */
uint64_t    i3d_sizeof_simplify_params(void);
uint64_t    i3d_sizeof_simplify_info(void);
/* Lindstrom's vertex clustering of the resident mesh: the vertices of each world-aligned cell of edge params->cell_size become one vertex
 * at the minimiser of the cell's summed, area-weighted face-plane quadrics (truncated pseudo-inverse around the members' mean; a
 * single-vertex cell keeps its vertex), faces that collapse or repeat an earlier face up to rotation are dropped, then the extraction's
 * degenerate faces and the vertices no face uses.  Deterministic: byte-equal to tests/mesh_simplify_ref.py.  The result replaces the
 * resident mesh that i3d_download_mesh reads (a further call simplifies it again); *info (may be NULL) gets the counts and the device time
 * per stage.  Fails, leaving the resident mesh and every other state as they were, without a resident mesh of the current grid, for a
 * cell_size that is not finite and > 0, and when a vertex's cell coordinate x / cell_size is not finite or outside int32.  A result
 * without faces is an empty resident mesh. */
int         i3d_simplify_mesh(I3DEngine* e, const I3DSimplifyParams* params, I3DSimplifyInfo* info);

/* ---- baking the keyframes' colour into a texture atlas of the resident mesh (DESIGN.md §6t) ---- */
uint64_t    i3d_sizeof_texture_params(void);
uint64_t    i3d_sizeof_texture_info(void);
/* texels_per_face 12, max_occlusion_distance 0.02, max_num_observations 5. */
void        i3d_default_texture_params(I3DTextureParams* p);
/* A texture atlas of the resident mesh, coloured from the keyframes.  Faces 2c and 2c+1 share square cell c of S x S texels (S =
 * params->texels_per_face), laid out row-major in the smallest square number of columns; every texel a face owns is coloured by
 * i3d_recompute_colors' rule at the 3-D point it maps to (observation weight at the face normal, top-K, weighted mean of the bilinear
 * colours), and a texel no frame observes gets the barycentric blend of the face's vertex colours.  The layout, the rounding of every
 * operation and the property that a bilinear lookup inside a face's UV triangle reads only texels of that face are in
 * i3d_texture.cuh.  pose_world_to_cam: float [F][12] (R row-major | t), or NULL for the engine's camera, as in i3d_recompute_colors.
 * The atlas and the per-corner UVs stay on the device until i3d_download_texture; *info (may be NULL) gets the counts and device time.
 * The bake also records which texels a keyframe observed (for i3d_decompose_texture's fallback count), a frame scan that stops at the
 * first observation; its device time is i3d_phase_ms("texture_observed"), not part of ms_bake.
 * The texture belongs to the resident mesh: an extraction, a successful simplification or a change of the voxel set drops it; a later
 * change of the camera or the frames does not update it.  Reads the mesh, frames, colour frames and camera only.  Fails, writing
 * nothing and leaving the previous texture, when world > 1, without a resident mesh with faces, without frames, camera or colour frames
 * of the current frame size, for texels_per_face outside [I3D_TEXTURE_MIN_TEXELS_PER_FACE, I3D_TEXTURE_MAX_TEXELS_PER_FACE],
 * max_num_observations outside [0, I3D_MAX_OBS], a max_occlusion_distance that is not finite, and an atlas side above
 * I3D_TEXTURE_MAX_SIDE. */
int         i3d_bake_texture(I3DEngine* e, const I3DTextureParams* params, const float* pose_world_to_cam, I3DTextureInfo* info);
/* The baked texture: rgb uint8 [H][W][3] in R, G, B order (W, H: info->atlas_width / atlas_height), uv float [F][3][2], per face corner
 * (u, v) as an OBJ reads them (v up).  Either pointer may be NULL.  Fails without a texture of the resident mesh. */
int         i3d_download_texture(I3DEngine* e, uint8_t* rgb, float* uv);

/* ---- albedo and shading of the baked texture, and relighting (DESIGN.md §6x) ---- */
uint64_t    i3d_sizeof_sh_lighting(void);
uint64_t    i3d_sizeof_intrinsic_texture_params(void);
uint64_t    i3d_sizeof_intrinsic_texture_info(void);
/* source I3D_SH_ESTIMATE, sh 0. */
void        i3d_default_sh_lighting(I3DShLighting* p);
/* lighting: i3d_default_sh_lighting; min_shading 0.05. */
void        i3d_default_intrinsic_texture_params(I3DIntrinsicTextureParams* p);
/* Splits the texture of the resident mesh (the last i3d_bake_texture) into albedo and shading under params->lighting.  Every texel a
 * face owns is taken at the bake's point P and face normal n; s = sh . basis(n) with the lighting's SH at P; the texel is lit iff n != 0
 * and s > min_shading, and then albedo = (c / 255) / s per channel of its baked colour c (the bake's fallback texels included), else 0.
 * The rounding of every operation is in i3d_texture.cuh.  The albedo [H][W][3] and shading [H][W] atlases stay on the device until
 * i3d_download_intrinsic_texture and are the source of I3D_RASTER_COLOR_RELIT; *info (may be NULL) gets the counts, the albedo range and
 * the device time.  The decomposition belongs to the texture: a new bake, or anything that drops the texture, drops it; a later lighting
 * estimate does not update it.  Fails, writing nothing and leaving the texture and any previous decomposition, when world > 1, without
 * a texture of the resident mesh, for a bad source, for I3D_SH_ESTIMATE without a lighting estimate of the current voxel set, for an
 * I3D_SH_GLOBAL sh that is not finite, and for a min_shading that is not finite or < 0. */
int         i3d_decompose_texture(I3DEngine* e, const I3DIntrinsicTextureParams* params, I3DIntrinsicTextureInfo* info);
/* The last decomposition: albedo float [H][W][3] (R, G, B), shading float [H][W] (0 where no face owns the texel or its normal is 0).
 * Either pointer may be NULL.  Fails without a decomposition of the resident mesh's texture. */
int         i3d_download_intrinsic_texture(I3DEngine* e, float* albedo, float* shading);
/* The lighting of I3D_RASTER_COLOR_RELIT (engine state; default I3D_SH_ESTIMATE, read when a rasterization runs).  Fails, keeping the
 * previous lighting, for a NULL lighting, a bad source and an I3D_SH_GLOBAL sh that is not finite. */
int         i3d_set_relight(I3DEngine* e, const I3DShLighting* lighting);

/* ---- distance from the resident mesh to a reference surface (DESIGN.md §6u) ---- */
uint64_t    i3d_sizeof_distance_params(void);
uint64_t    i3d_sizeof_distance_info(void);
/* samples_per_edge 2, max_distance 0.01, cell_size 0 (automatic), thresholds 0.0002, 0.0005, 0.001. */
void        i3d_default_distance_params(I3DDistanceParams* p);
/* Copies a reference mesh xyz float [V][3], faces int32 [F][3] to the device, replacing the previous one.  It stays through grid,
 * frame and mesh changes.  Fails, keeping the previous reference, for V <= 0, F <= 0, NULL buffers, a vertex index outside [0, V), a
 * coordinate that is not finite, V > INT_MAX or 3 F > INT_MAX. */
int         i3d_upload_reference_mesh(I3DEngine* e, int64_t V, const float* xyz, int64_t F, const int32_t* faces);
/* Distances between the resident mesh A (the last extraction or simplification) and the reference mesh B: every face of either mesh is
 * sampled at the centroids of its L^2 congruent sub-triangles, weighted by area / L^2, and each sample gets the nearest face of the
 * other mesh within max_distance (the lexicographic minimum of (float d^2, face id) over all faces, so equal distances go to the
 * lowest face id); every vertex of A gets its nearest face of B.  *info gets per direction the sample counts, area-weighted mean, RMS
 * and maximum distance, the area fraction within each threshold, the grid used and the device time per stage, and precision, recall
 * and F-score per threshold.  The rounding of every operation is stated in i3d_distance.cuh; every result is bit-identical from run to
 * run.  Reads the meshes only.  Fails, leaving the resident mesh, its texture and the previous results as they were, when world > 1,
 * without a resident mesh with faces, without a reference mesh, for samples_per_edge outside [1, 16], a max_distance that is not
 * finite and > 0, a cell_size that is negative or not finite, num_thresholds outside [0, 8], thresholds that are not finite, not
 * ascending or above max_distance, and a search grid above I3D_DISTANCE_MAX_CELLS cells or I3D_DISTANCE_MAX_CELL_ENTRIES entries. */
int         i3d_surface_distance(I3DEngine* e, const I3DDistanceParams* params, I3DDistanceInfo* info);
/* The per-vertex results of the last i3d_surface_distance: vertex_distance float [V] (metres, +inf when no face of the reference is
 * within max_distance) and vertex_face int32 [V] (-1 then), V = info->num_vertices.  Either pointer may be NULL.  Fails before the
 * first successful call. */
int         i3d_download_surface_distance(I3DEngine* e, float* vertex_distance, int32_t* vertex_face);
/* Tests: keep the per-sample (d^2, face) of later i3d_surface_distance calls (on != 0), and read those of the last call: direction
 * 0 = resident -> reference, 1 = reference -> resident; d2 float [side[direction].num_samples] (+inf when unmatched), face int32 (-1). */
int         i3d_debug_set_keep_distance_samples(I3DEngine* e, int on);
int         i3d_debug_get_distance_samples(I3DEngine* e, int direction, float* d2, int32_t* face);

/* ---- registering the reference mesh to the resident mesh: point-to-plane ICP (DESIGN.md §6aa) ---- */
uint64_t    i3d_sizeof_register_params(void);
uint64_t    i3d_sizeof_register_info(void);
/* samples_per_edge 1, stages {0.016, 0.008, 0.004} m with 10 iterations each, min_normal_cos 0.5, min_correspondences 100, cell_size 0. */
void        i3d_default_register_params(I3DRegisterParams* p);
/* Estimates the rigid T (R row-major | t, 12 doubles) with x_A = R x_B + t that maps the reference mesh B onto the resident mesh A, by
 * point-to-plane Gauss-Newton from T_init (NULL = identity): the samples of A (i3d_surface_distance's, weighted by area / L^2) are moved
 * by T^-1 and each is paired with the nearest face of B within the stage's max_distance; a row needs both unit face normals non-zero
 * and dot(n_A, n_B) >= min_normal_cos.  The stages run in order with no early stop, then one more system is formed at the final pose;
 * the 6 x 6 solve and the update are the tracker's, with its statuses.  Every result is bit-identical from run to run and does not depend
 * on cell_size; the rounding of every operation is stated in i3d_register.cuh.  Writes T_out and *info (may be NULL) only: the reference,
 * the resident mesh, its texture and the last distance results stay as they were.  Fails, writing nothing, when world > 1, without a
 * resident mesh with faces, without a reference mesh, for a parameter out of its range, a T_init that is not finite or not a rotation
 * (max |R^T R - I| > 1e-5 or det R < 0), a NULL T_out, and a search grid above the caps of i3d_surface_distance. */
int         i3d_register_reference_mesh(I3DEngine* e, const I3DRegisterParams* params, const double* T_init, double* T_out, I3DRegisterInfo* info);
/* Moves the reference mesh on the device: every vertex x <- float(((R0 x0 + R1 x1) + R2 x2) + t), per row of R, in double from the float
 * x.  i3d_surface_distance and i3d_grid_from_mesh (reference source) then use the moved mesh; the last distance results are kept.  Fails,
 * changing nothing, without a reference mesh and for a T that is not finite or not a rotation (as above). */
int         i3d_transform_reference_mesh(I3DEngine* e, const double* T);
/* Tests: the systems of the last i3d_register_reference_mesh, in the order they were formed (the first at T_init, the last the one
 * without a solve at the final pose); n = their number.  systems double [n][31]: the 29 sums of the tracker's layout (21 upper-triangle
 * entries of sum w J^T J, 6 of sum w J^T r, sum w r^2, rows), then sum w (for the first and the last system only, else 0) and 0;
 * poses double [n][12]: T^-1 at which each was formed; faces int32 [F L^2]: per sample the nearest face of B at T_init (-1 when none or
 * for a zero-area face).  Any pointer may be NULL.  Fails before the first successful call. */
int         i3d_debug_get_register_systems(I3DEngine* e, int32_t* n, double* systems, double* poses, int32_t* faces);

/* ---- the voxel grid from a triangle mesh: narrow-band signed distance (DESIGN.md §6v) ---- */
uint64_t    i3d_sizeof_grid_from_mesh_params(void);
uint64_t    i3d_sizeof_grid_from_mesh_info(void);
/* source I3D_GRID_FROM_MESH_REFERENCE, voxel_size 0.002, band 3, cell_size 0 (automatic). */
void        i3d_default_grid_from_mesh_params(I3DGridFromMeshParams* p);
/* Replaces the voxel set by the narrow-band signed distance field of a triangle mesh on the lattice c * voxel_size: every voxel with a
 * face within b = band * voxel_size gets the nearest face (the lexicographic minimum of (float d^2, face id), as i3d_surface_distance
 * finds it), |sdf| = sqrt(d^2) and the sign of dot(p - q, N), N the angle-weighted pseudonormal of the feature of the face the closest
 * point q lies on, over vertices welded by exact position.  A voxel is dropped when N = 0, when dot = 0 at d > 0, and when the feature
 * lies on the mesh's boundary and |cos(p - q, N)| < I3D_GRID_FROM_MESH_RIM_COS.  Voxels come in canonical 8^3-brick-major order with
 * sdf0 = sdf, albedo 0.6, weight 1 and colour 0 (i3d_recompute_colors colours them); voxel_size and truncation (5 voxels) are set as
 * i3d_fusion_finish sets them.  The rounding of every operation is stated in i3d_grid_from_mesh.cuh; the result does not depend on
 * cell_size and is bit-identical from run to run.  On success everything derived from the voxel set is forgotten (as after a pruning),
 * and the frames, camera, sensor store, reference mesh and any fusion in progress stay.  *info (may be NULL) gets the counts and the
 * device time per stage.  Fails, changing nothing, when world > 1, without the source mesh or with one without faces, for a bad
 * source, a voxel_size that is not finite and > 0, a band outside (0, 16], a cell_size that is negative or not finite, a lattice
 * coordinate outside +-(2^20 - 8), a search grid above the caps of i3d_surface_distance, more than I3D_GRID_FROM_MESH_MAX_PAIRS
 * (face, brick) pairs or I3D_GRID_FROM_MESH_MAX_VOXELS candidate voxels, and when no voxel is emitted. */
int         i3d_grid_from_mesh(I3DEngine* e, const I3DGridFromMeshParams* params, I3DGridFromMeshInfo* info);
/* Tests: per voxel of the last successful i3d_grid_from_mesh (in its order), the nearest face int32 and the I3D_FEATURE_* of the
 * closest point int8.  Either pointer may be NULL.  Fails before the first successful call. */
int         i3d_debug_get_grid_from_mesh_voxels(I3DEngine* e, int32_t* face, int8_t* feature);

/* ---- rasterizing the resident mesh into the keyframes and into new views (DESIGN.md §6w) ---- */
uint64_t    i3d_sizeof_raster_params(void);
uint64_t    i3d_sizeof_raster_camera(void);
uint64_t    i3d_sizeof_raster_stats(void);
uint64_t    i3d_sizeof_raster_info(void);
/* every plane, vertex colours. */
void        i3d_default_raster_params(I3DRasterParams* p);
/* Rasterizes the resident mesh (the last extraction or simplification) into the frames ids[0..n) with the camera of the frame scans at
 * the current pyramid level: W x H of the installed frames, the float R | t of i3d_render_keyframes and its intrinsics * pyr_scale with
 * the five distortion coefficients.  Per pixel the nearest face of either orientation along the pixel's undistorted ray (a watertight
 * ray-triangle test; equal depths go to the lowest face id), with the requested planes (I3D_RASTER_*) and the colour of
 * params->color_source: the vertex colours, the texture of i3d_bake_texture, or its decomposition relit (I3D_RASTER_COLOR_RELIT: the
 * bilinear albedo times the shading at the face normal under the lighting of i3d_set_relight).  stats[n] (may be NULL) compares each view with its
 * frame's depth and, with a colour source, its colour frame; *info (may be NULL) gets the counts and the device time per stage.  The
 * rounding of every operation is stated in i3d_raster.cuh; the planes and statistics are bit-identical from run to run and do not depend
 * on the batch.  The planes belong to the resident mesh and stay for i3d_download_raster: an extraction, a successful simplification, a
 * change of the voxel set or of the frames drops them; a later camera change does not update them.  Reads the mesh, texture, frames and
 * camera only.  Fails, writing nothing and leaving the previous planes, when world > 1, without a resident mesh with faces, for n <= 0,
 * n > 65535, a NULL ids or an id out of [0, F), without frames or camera, for intrinsics (after pyr_scale) that are not finite with fx,
 * fy > 0, distortion that is not finite, a bad plane mask or colour source, the texture source without a texture of the resident mesh,
 * the relit source without a decomposition of that texture or, under I3D_SH_ESTIMATE, without a lighting estimate of the current voxel
 * set, and a colour source without colour frames of the current frame size.  Device time: i3d_phase_ms("raster"), of which "raster_bin" (ray
 * table and tile boxes), "raster_faces" (binning and triangle tests) and "raster_shade"; i3d_phase_count("raster_tests") = the
 * ray-triangle tests. */
int         i3d_rasterize_keyframes(I3DEngine* e, int32_t n, const int32_t* ids, const I3DRasterParams* params, I3DRasterStats* stats,
                                    I3DRasterInfo* info);
/* The same into n new views of *camera (width x height, its own intrinsics and distortion) at pose_world_to_cam float [n][12] (R
 * row-major | t, world -> camera); no statistics.  Fails as i3d_rasterize_keyframes where it applies, and for a NULL camera or pose, a
 * pose entry that is not finite, and a width or height outside [1, I3D_RASTER_MAX_SIDE]. */
int         i3d_rasterize_views(I3DEngine* e, int32_t n, const I3DRasterCamera* camera, const float* pose_world_to_cam,
                                const I3DRasterParams* params, I3DRasterInfo* info);
/* The planes of the last rasterization, [n][H][W]: depth float, face int32, bary float [2], normal float [3], rgb uint8 [3].  Any pointer
 * may be NULL.  Fails for a plane that was not rendered and when no rasterization of the resident mesh exists. */
int         i3d_download_raster(I3DEngine* e, float* depth, int32_t* face, float* bary, float* normal, uint8_t* rgb);
/* on = 1 (default): faces are binned to 8 x 8 pixel tiles by their padded projected box; 0: every face goes to every tile and every
 * pixel is tested.  The results are the same. */
int         i3d_debug_set_raster_binning(I3DEngine* e, int on);
/* views > 0: a rasterization runs in passes of at most that many views (the passes a large call splits into); 0 (default): as many
 * as 2^27 (view, pixel) keys allow.  The results are the same.  Fails for views < 0. */
int         i3d_debug_set_raster_batch(I3DEngine* e, int views);

/* ---- rendering the surface into the keyframes (DESIGN.md §6m) ---- */
uint64_t    i3d_sizeof_render_params(void);
uint64_t    i3d_sizeof_render_stats(void);
/* sdf_source 1, every plane, photometric pairs on. */
void        i3d_default_render_params(I3DRenderParams* p);
/* Ray-casts the zero level set of params->sdf_source into the frames ids[0..n) of the resident camera state at the current pyramid level:
 * W x H of the installed frames, the float R | t of the frame scans and their intrinsics * pyr_scale with the five distortion
 * coefficients.  stats[n] (may be NULL) compares each view with its frame's depth and luminance.  The requested planes stay resident for
 * i3d_download_render.  Reads the grid, camera, SH and frames only.  Fails, writing nothing, without grid, frames or camera, for n <= 0,
 * n > 65535 or an id out of [0, F), a bad source or plane mask, shading / intensity planes or photometric pairs without per-voxel SH,
 * intrinsics (after pyr_scale) that are not finite with fx, fy > 0, distortion that is not finite, and for world > 1.  A frame whose pose
 * is not finite renders as a view without hits.  Device time: i3d_phase_ms("render"), of which the occupancy bitmap (built on the first
 * render after a voxel-set change)
 * is i3d_phase_ms("render_bricks"); lattice samples evaluated: i3d_phase_count("render_samples"). */
int         i3d_render_keyframes(I3DEngine* e, int32_t n, const int32_t* ids, const I3DRenderParams* params, I3DRenderStats* stats);
/* The planes of the last render, float32 [n][H][W] (normal [n][H][W][3]).  Any pointer may be NULL.  Fails for a plane that was not
 * rendered, and when no render of the current voxel set and frames exists.  The planes are those of the state at render time: a later
 * i3d_set_camera, i3d_upload_voxel_params or i3d_gn_iteration neither updates nor drops them (render again to see the new state), as the
 * resident mesh of i3d_extract_mesh; a change of the voxel set or of the frames drops them. */
int         i3d_download_render(I3DEngine* e, float* depth, float* normal, float* albedo, float* shading, float* intensity);

/* ---- tracking sensor frames against the surface: point-to-plane ICP over the depth pyramid (DESIGN.md §6n) ---- */
/* Frames tracked per device pass: bounds the scratch memory (I3D_TRACK_CHUNK prediction, pyramid and normal planes at depth size). */
#define I3D_TRACK_CHUNK 32
uint64_t    i3d_sizeof_track_params(void);
uint64_t    i3d_sizeof_track_info(void);
/* sdf_source 0, 3 levels, iterations {10, 5, 4, 0}, max_distance 0.05 m, min_normal_cos cos(20 deg), min_correspondences 100. */
void        i3d_default_track_params(I3DTrackParams* p);
/* Frame-to-model tracking of the stored sensor frames ids[0..n) (distinct ids) against params->sdf_source of the current grid.  Per frame:
 * the surface rendered at the input pose with the store's depth camera (the prediction), the depth pyramid of the stored depth, and
 * Gauss-Newton iterations of point-to-plane ICP, coarsest level first, every iteration enqueued without host synchronisation.
 * pose_in / pose_out: world -> camera, double [n][12] (R row-major | t), the Rt layout of fusion and render; info[n] may be NULL.
 * Reads the grid, the store and the renderer's voxel box; writes only its own buffers, pose_out and info.  A frame's result does not depend
 * on the other frames of the call.  Fails, writing nothing, without grid or stored frames, for n <= 0 or n > 65535, an id out of range or
 * repeated, a non-finite input pose, num_levels outside 1..4 or a level built from a level under 3 px, negative iterations, max_distance
 * not finite and > 0, min_normal_cos outside [-1, 1], min_correspondences < 6, a bad sdf_source, and world > 1.
 * Device time: i3d_phase_ms("track") for the call, of which "track_predict", "track_pyramid" and "track_icp";
 * i3d_phase_count("track_correspondences") = rows of every evaluated system. */
int         i3d_track_sensor_frames(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params,
                                    double* pose_out, I3DTrackInfo* info);
/* Parity hook: sums [n][29] = the last evaluated system of each frame of the last call (21 upper-triangle entries of J^T J row by row,
 * 6 of J^T r, sum r^2, rows) and pose_cam_to_world [n][12] = its pose state (R row-major | t, camera -> world) after the last solve.
 * Either pointer may be NULL.  Fails before a tracking call. */
int         i3d_debug_get_track_system(I3DEngine* e, double* sums, double* pose_cam_to_world);
/* Parity hook: the planes of the last pass (the last I3D_TRACK_CHUNK frames or fewer) of the last call, for the frames of that pass:
 * depth [m][H_l][W_l] and camera-frame normals [m][H_l][W_l][3] of pyramid level `level`, the prediction depth [m][H][W] and world
 * normals [m][H][W][3], and mask uint8 [m][H][W] (1 = a correspondence of the last level-0 system).  Any pointer may be NULL.  m is
 * returned in *frames (may be NULL).  Fails before a tracking call and for a level that call did not build. */
int         i3d_debug_get_track_planes(I3DEngine* e, int32_t level, float* depth, float* normal, float* pred_depth, float* pred_normal,
                                       uint8_t* mask, int32_t* frames);

/* ---- tracking against the fusion in progress, and dense RGB-D odometry (DESIGN.md §6o) ---- */
/* i3d_track_sensor_frames with the fusion volume in progress as the model: the prediction is marched through the fusion's own table (a
 * cube is valid when its 8 corners exist with weight != 0; the value is the trilinear blend of the float Voxel::sdf) inside the box of the
 * voxels with weight > 0, whose brick bitmap is rebuilt here.  Equal byte for byte to i3d_fusion_finish with correct_sdf_iterations = 0
 * followed by i3d_track_sensor_frames(sdf_source 0).  params->sdf_source must be 0.  Writes only its own buffers, pose_out and info: the
 * fusion volume, the grid, the renderer's state and the resident mesh and render are left as they were.  Fails, writing none of those,
 * without a fusion in progress, when no voxel has weight > 0, and for every refusal of i3d_track_sensor_frames except "no grid".
 * Device time as there, plus i3d_phase_ms("track_bricks") for the box and bitmap. */
int         i3d_fusion_track_sensor_frames(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params,
                                           double* pose_out, I3DTrackInfo* info);
/* Dense frame-to-model odometry: the stored frames ids[0..n) (repeats allowed), in list order, each tracked against the fusion in progress
 * and then integrated into it.  Per frame:
 *   1. the guess: pose_first (world -> camera [12]) for ids[0] when it is not NULL, which resets the motion state; otherwise the motion
 *      state the fusion keeps (i3d_fusion_begin and every i3d_fusion_integrate* call clear it).  With two previous poses the guess is the
 *      constant-velocity one, in double with camera -> world poses T: T(k) = T(k-1) . (T(k-2)^-1 . T(k-1)); with one, T(k-1).
 *   2. no voxel with weight > 0: the frame is integrated at the guess, untracked (status I3D_TRACK_ANCHORED).
 *   3. otherwise i3d_fusion_track_sensor_frames of that frame from the guess; at status I3D_TRACK_OK the frame is integrated at the
 *      tracked pose (the float camera -> world and world -> camera of the double pose).  At any other status it is not integrated,
 *      pose_out is the guess and the velocity becomes zero at the last integrated pose (the guess when the state has none).
 * pose_out [n][12] world -> camera, info[n] may be NULL.  Calls chain: n frames in one call or in several with pose_first = NULL after
 * the first give the same bytes.  Fails, leaving the fusion in progress and every state as it was, for the refusals of
 * i3d_fusion_track_sensor_frames (repeated ids and n > 65535 allowed), a non-finite pose_first, and pose_first = NULL without a motion
 * state.  A failure while fusing ends the fusion as i3d_fusion_integrate_sensor does.  Time: i3d_phase_ms("odometry") is the call's host
 * wall time, of which the device times "odometry_predict" (box, bitmap, prediction) and "odometry_icp" (pyramid and ICP) and the fusion
 * phases; i3d_phase_count("odometry_correspondences") = rows of every evaluated system. */
int         i3d_fusion_track_and_integrate_sensor(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_first,
                                                  const I3DTrackParams* params, double* pose_out, I3DTrackInfo* info);

/* ---- tracking with colour as well as depth: a photometric term (DESIGN.md §6p) ---- */
uint64_t    i3d_sizeof_track_color_params(void);
uint64_t    i3d_sizeof_track_color_info(void);
/* weight {0.05, 0.05, 0.05, 0.05}, max_color_diff 0.1, min_color_gradient 0.01 (the best of the weights measured on C2, DESIGN.md §6p). */
void        i3d_default_track_color_params(I3DTrackColorParams* p);
/* The three tracking calls with a photometric term added to every system: per level the prediction pixels (2^l u, 2^l v) with a hit give
 * a world point q and the model intensity I_m (the trilinear blend of the voxel colours' intensities at the hit), the residual is
 * I_f(pi(R^T (q - t))) - I_m against the stored colour frame's intensity in the depth camera at level l, and the system solved is
 * A_depth + lambda_l^2 A_colour, b likewise; the row count, sum r^2 and every status keep their depth-only meaning.  With every weight 0
 * the results are the bytes of the depth-only call.  color_info[n] (may be NULL): the photometric rows and sum r^2 of the first and the
 * last evaluated system.  Fail, writing nothing, for every refusal of the depth-only call, NULL color params, a weight that is negative or
 * not finite, max_color_diff not finite and > 0, and min_color_gradient negative or not finite.  Device time as the depth-only call, plus
 * i3d_phase_ms("track_color") (intensity pyramid and gradients); i3d_phase_count("track_photo_correspondences") = photometric rows of
 * every evaluated system; with i3d_debug_set_kernel_timers(e, 1) also "track_photo_rows". */
int         i3d_track_sensor_frames_rgbd(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params,
                                         const I3DTrackColorParams* color, double* pose_out, I3DTrackInfo* info, I3DTrackColorInfo* color_info);
int         i3d_fusion_track_sensor_frames_rgbd(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const I3DTrackParams* params,
                                                const I3DTrackColorParams* color, double* pose_out, I3DTrackInfo* info,
                                                I3DTrackColorInfo* color_info);
int         i3d_fusion_track_and_integrate_sensor_rgbd(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_first,
                                                       const I3DTrackParams* params, const I3DTrackColorParams* color, double* pose_out,
                                                       I3DTrackInfo* info, I3DTrackColorInfo* color_info);
/* Parity hook: the planes of the last pass of the last _rgbd call, for the frames of that pass: model_intensity [m][H][W] (0 without a
 * hit), and at pyramid level `level` the frame intensity, grad_x and grad_y [m][H_l][W_l].  Any pointer may be NULL; m in *frames.  Fails
 * when the last tracking call had no photometric term and for a level it did not build. */
int         i3d_debug_get_track_color_planes(I3DEngine* e, int32_t level, float* model_intensity, float* intensity, float* grad_x,
                                             float* grad_y, int32_t* frames);
/* Parity hook: sums [n][29] = the photometric values of the last evaluated system of each frame of the last _rgbd call, in the layout of
 * i3d_debug_get_track_system, unweighted.  Fails when the last tracking call had no photometric term. */
int         i3d_debug_get_track_color_system(I3DEngine* e, double* sums);

/* ---- the photometric term against a reference frame's image (DESIGN.md §6q) ---- */
/* i3d_default_track_color_params with weight {0.01, 0.01, 0.01, 0.01}: the best of the weights measured with the reference model on C2
 * (DESIGN.md §6q). */
void        i3d_default_track_color_ref_params(I3DTrackColorParams* p);
/* The _rgbd calls with the model intensity taken from a reference frame instead of the voxel colours: the prediction is marched without
 * colour, and at level l the model value of prediction pixel (2^l u, 2^l v) with a hit is the stored frame ref_ids[k]'s level-l intensity
 * (the frame's own rules: intensity in the depth camera, then pyrDown), bilinear at the projection of the model point q with ref_pose[k]
 * (world -> camera [12], R row-major | t, used in float), when the projection lies in [1, W_l - 2) x [1, H_l - 2) and the reference's
 * level-l depth at the rounded pixel is > 0 and within max_distance of q's depth there; else no photometric row.  A frame may be its own
 * reference.  Fail, writing nothing, for every refusal of the matching _rgbd call, NULL ref_ids or ref_pose, a reference id out of range
 * and a non-finite reference pose.  Device time as the _rgbd call, plus i3d_phase_ms("track_reference") (the references' pyramids and
 * model planes); with i3d_debug_set_kernel_timers(e, 1) also "track_ref_model". */
int         i3d_track_sensor_frames_rgbd_ref(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const int32_t* ref_ids,
                                             const double* ref_pose, const I3DTrackParams* params, const I3DTrackColorParams* color,
                                             double* pose_out, I3DTrackInfo* info, I3DTrackColorInfo* color_info);
int         i3d_fusion_track_sensor_frames_rgbd_ref(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_in, const int32_t* ref_ids,
                                                    const double* ref_pose, const I3DTrackParams* params, const I3DTrackColorParams* color,
                                                    double* pose_out, I3DTrackInfo* info, I3DTrackColorInfo* color_info);
/* Dense odometry with the reference model: each frame's reference is the last frame this loop integrated (anchored or tracked), at the
 * camera -> world pose it was integrated with.  The reference lives in the fusion beside the motion state and is cleared where that is
 * (i3d_fusion_begin, every i3d_fusion_integrate* call, a pose_first) and by i3d_sensor_frames_begin, whose new store no longer holds it;
 * a frame without one is tracked on depth alone, with zero color_info.
 * Timed as the _rgbd loop; the reference work counts as "odometry_icp". */
int         i3d_fusion_track_and_integrate_sensor_rgbd_ref(I3DEngine* e, int32_t n, const int32_t* ids, const double* pose_first,
                                                           const I3DTrackParams* params, const I3DTrackColorParams* color, double* pose_out,
                                                           I3DTrackInfo* info, I3DTrackColorInfo* color_info);
/* Parity hook: the planes of the last pass of the last _ref call at pyramid `level`, compact [m][H_l][W_l] each: the model value (the quiet
 * NaN where there is none), and the references' intensity and depth.  Any pointer may be NULL; m in *frames.  Fails when the last
 * tracking call was not a _ref call with a reference and for a level it did not build.  After a _ref call
 * i3d_debug_get_track_color_planes refuses a non-NULL model_intensity. */
int         i3d_debug_get_track_reference_planes(I3DEngine* e, int32_t level, float* model, float* ref_intensity, float* ref_depth,
                                                 int32_t* frames);

/* ---- locally normalised intensity for the reference model (DESIGN.md §6r) ---- */
/* The largest norm_radius of I3DTrackColorParams. */
#define I3D_TRACK_MAX_NORM_RADIUS 8
/* With color->norm_radius = r > 0 the three _ref calls compare locally normalised intensity: every level of the frame's and of the
 * reference's intensity pyramid (each level still the pyrDown of the raw level above) becomes (I - mu) / sqrt(max(m2 - mu^2, 0) +
 * norm_eps^2), mu and m2 the float32 mean of I and I^2 over the (2r+1)^2 window clipped to the image, and exactly 0 where that window is
 * constant.  A gain and offset constant over the window cancel, so per-frame exposure and white-balance changes that vary slowly across
 * the image no longer bias the residual.  Everything after the planes is unchanged; max_color_diff, min_color_gradient and the residuals
 * of color_info are in normalised units, and i3d_debug_get_track_color_planes / i3d_debug_get_track_reference_planes return the
 * normalised planes the rows read.  norm_radius 0 gives the bytes of today's _ref calls.  The _ref calls fail, writing nothing, for
 * norm_radius < 0 or > I3D_TRACK_MAX_NORM_RADIUS and, with norm_radius > 0, norm_eps not finite or <= 0; the _rgbd calls (voxel model,
 * whose model plane has holes) fail for norm_radius != 0.  With i3d_debug_set_kernel_timers(e, 1) also "track_local_norm". */
/* i3d_default_track_color_ref_params with the LNI parameters measured on C2 (DESIGN.md §6r). */
void        i3d_default_track_color_lni_params(I3DTrackColorParams* p);

/* ---- keyframe selection and the RGB-D image pyramid: the inputs of fusion and refinement (DESIGN.md §6i) ---- */
/* Frames scored per device pass by i3d_keyframe_scores: bounds its scratch memory (I3D_KEYFRAME_CHUNK * W * H * 3 bytes). */
#define I3D_KEYFRAME_CHUNK 32
/* KeyframeSelection::add / estimateBlur (src/keyframe_selection.cpp:64-70, 219-310) for F frames: bgr uint8 [F][H][W][3] interleaved
 * B,G,R; scores[F] = the Crete-2007 no-reference blur score (1 = sharp), NaN for a frame without vertical variation as in the reference.
 * A frame's score depends only on its own pixels (not on F or on the other frames).  Fails for F <= 0 or frames under 5 px on an axis.
 * Device time of the last call: i3d_phase_ms("keyframe_scores"); passes: i3d_phase_count("keyframe_chunks"). */
int         i3d_keyframe_scores(I3DEngine* e, int32_t F, int32_t W, int32_t H, const uint8_t* bgr, double* scores);
/* The level-0 keyframes (Pyramid::create's inputs, src/rgbd/pyramid.cpp:59-79) into a device-resident frame store: bgr uint8 [F][H][W][3],
 * depth float metres [F][H][W], lum float [F][H][W] = Pyramid::intensity(0), or NULL to compute it from bgr (float B,G,R / 255, then
 * (B 0.114 + G 0.587) + R 0.299).  The store replaces any previous one; the frames the engine is using are left alone. */
int         i3d_upload_rgbd_frames(I3DEngine* e, int32_t F, int32_t W, int32_t H, const uint8_t* bgr, const float* depth, const float* lum);
/* Builds Pyramid::intensity(lvl) (cv::pyrDown chain) and Pyramid::depth(lvl) (downsampleDepth chain) of every stored frame on the device and
 * installs them exactly as i3d_upload_frames(F, W_lvl, H_lvl, lum, depth, 2^-lvl) would (same camera, iteration and colour invalidation);
 * at lvl 0 the stored colours also become resident as i3d_upload_color_frames would make them.  *W_out / *H_out (may be NULL) get the
 * level's size.  Fails without a store, for lvl < 0, and when a level on the way is under 3 px on an axis.
 * Device time of the last call: i3d_phase_ms("frames_level"). */
int         i3d_use_rgbd_level(I3DEngine* e, int32_t lvl, int32_t* W_out, int32_t* H_out);

/* ---- the sensor store: the raw RGB-D sequence on the device, uploaded once (DESIGN.md §6l) ---- */
/* Starts an empty store of `capacity` frames (Sensor::depth(i) / Sensor::color(i)) and allocates its device memory for all of them:
 * depth float metres [depth_cam.height][depth_cam.width], already range-thresholded as i3d_fusion_integrate takes it, and colour uint8
 * [color_cam.height][color_cam.width][3] interleaved B,G,R.  Replaces any previous store; the frame store of i3d_upload_rgbd_frames is a
 * separate one and is left alone.  Clears the reference of the _ref odometry (a frame of the replaced store); the next frame of that loop
 * is tracked on depth alone.  Fails for a camera without a positive size, finite intrinsics and fx, fy > 0, and for capacity <= 0. */
int         i3d_sensor_frames_begin(I3DEngine* e, const I3DFusionCamera* depth_cam, const I3DFusionCamera* color_cam, int32_t capacity);
/* Appends F frames (ids i3d_sensor_num_frames(), +1, ...): depth [F][...] and bgr [F][...] in the layouts above.  Fails without a store,
 * for F <= 0 and beyond the capacity. */
int         i3d_sensor_frames_add(I3DEngine* e, int32_t F, const float* depth, const uint8_t* bgr);
/* Frames in the store (0 without one). */
int32_t     i3d_sensor_num_frames(const I3DEngine* e);
/* i3d_keyframe_scores of every stored frame, read from the store: scores[i3d_sensor_num_frames()], byte-equal to i3d_keyframe_scores of
 * the same frames.  Fails without stored frames and for colour frames under 5 px on an axis.  Device time: i3d_phase_ms("keyframe_scores"). */
int         i3d_sensor_keyframe_scores(I3DEngine* e, double* scores);
/* i3d_fusion_integrate of the stored frames ids[0..n), in list order, with the store's two cameras; pose_cam_to_world and
 * pose_world_to_cam are [n][12] as there.  The store is only read.  Fails, leaving the fusion in progress, without a fusion in progress,
 * without stored frames, for n <= 0 and for an id out of range; a failure while fusing ends the fusion as i3d_fusion_integrate does. */
int         i3d_fusion_integrate_sensor(I3DEngine* e, int32_t n, const int32_t* ids, const float* pose_cam_to_world,
                                        const float* pose_world_to_cam);
/* The per-keyframe part of Intrinsic3D::init (src/refinement/intrinsic3d.cpp:176-190) for the stored frames ids[0..n) (any order, repeats
 * allowed): the colour, resizeDepth of the depth to the colour camera (src/rgbd/processing.cpp:129-183; a copy when the sizes agree) and
 * the level-0 intensity fill the frame store exactly as i3d_upload_rgbd_frames(n, color W, color H, bgr[ids], resizeDepth(depth[ids]), NULL)
 * would; i3d_use_rgbd_level then works as after that call.  Fails without stored frames, for n <= 0 and for an id out of range, leaving
 * both stores as they were.  Device time: i3d_phase_ms("sensor_select"), of which k_resize_depth is i3d_phase_ms("resize_depth"). */
int         i3d_select_rgbd_frames(I3DEngine* e, int32_t n, const int32_t* ids);

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
/* PCG iterate x[U] and search direction p[U] (Jacobi-scaled unknown space) as the last LM trial's solve left them.  Any pointer may be
 * NULL. */
int         i3d_debug_get_pcg_vectors(I3DEngine* e, float* x, float* p);
/* normal-equation pieces of the last iteration (build_only = 1 is enough), unknown space [U = 2n + 6F + 9]: b[U] = J'^T f (Jacobi
 * scaled gradient), s[U] (Jacobi column scale, 0 for fixed unknowns), jtj[U] = s^2 * column norm^2, and the raw (unweighted by the
 * type weight, unscaled) E_g camera sums cam_acc[33F + 43]: per frame 6 gradient (sum w_raw r J), 6 column norms, the upper 6x6
 * triangle row by row (21); then 9 gradient, 9 column norms of intrinsics | distortion, the upper 4x4 (10) and 5x5 (15) triangles.
 * Any pointer may be NULL. */
int         i3d_debug_get_normal_equations(I3DEngine* e, float* b, float* s, float* jtj, float* cam_acc);
/* q[U] = S (J^T W J) S v for the rows of the last iteration (all four terms, no D^2 term): the raw operator output of the production
 * k_eg_apply + k_op_partial pair times s, in float.  Leaves nothing behind that a following i3d_gn_iteration reads.  Single GPU only. */
int         i3d_debug_apply_operator(I3DEngine* e, const float* v, float* q);
/* Voxels of the fusion volume in progress (allocated ones included, integrated or not); 0 outside a fusion. */
int64_t     i3d_debug_fusion_num_voxels(const I3DEngine* e);
/* The fusion volume in progress in canonical order (see i3d_fusion_finish): xyz[3n], sdf[n] (Voxel::sdf, float), weight[n],
 * rgb[3n] (r,g,b).  Any pointer may be NULL.  Fusion stage timings: i3d_phase_ms("fusion_prep" | "fusion_alloc" |
 * "fusion_integrate" | "fusion_correct" | "fusion_finish"); i3d_phase_count("fusion_growths" | "fusion_sweeps"). */
int         i3d_debug_get_fusion_volume(I3DEngine* e, int32_t* xyz, float* sdf, float* weight, uint8_t* rgb);
/* The frames of the current level as the device holds them: lum[F][H][W], depth[F][H][W], bgr[F][H][W][3] (fails when asked for colours
 * that are not resident at this size).  Any pointer may be NULL. */
int         i3d_debug_get_frames(I3DEngine* e, float* lum, float* depth, uint8_t* bgr);
/* on = 1 (default): i3d_render_keyframes jumps over empty 8^3 bricks; 0: it evaluates every lattice sample.  The results are the same. */
int         i3d_debug_set_render_skip(I3DEngine* e, int on);

#ifdef __cplusplus
}
#endif
#endif /* I3D_C_API_H_ */
