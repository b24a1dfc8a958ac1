/*
 * i3d_types.h — plain-C parameter / result structs shared by the H100 engine
 * C-ABI (include/i3d_c_api.h) and by the CPU oracle (oracle/oracle_api.h).
 *
 * Field meanings follow the reference (paths relative to the NVlabs/intrinsic3d
 * tree, libintrinsic3d/ = L/):
 *   - cost-type ids 0..3 = E_g, E_r, E_s, E_a as set in
 *     L/src/refinement/optimizer.cpp:140-143
 *   - solver options = Ceres 2.1.0 defaults the reference leaves untouched
 *     (L/src/refinement/nls_solver.cpp:300-337 sets only max_num_iterations,
 *     CGNR, num_threads).
 */
#ifndef I3D_TYPES_H_
#define I3D_TYPES_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define I3D_NUM_COST_TYPES 4
#define I3D_MAX_OBS 8          /* upper bound for num_observations (reference default 5) */
#define I3D_EG_COLS 29         /* 10 sdf + 4 albedo + 6 pose + 4 intrinsics + 5 distortion */
#define I3D_MAX_LM_STEPS 64    /* per-trial bookkeeping slots in I3DIterInfo */

/* Parameters of ONE Gauss-Newton (outer) iteration of Optimizer::optimize
 * (L/src/refinement/optimizer.cpp:119-171). The host shim computes the ramped
 * lambdas (L/include/nv/refinement/cost.h:130-143) and the term switches. */
typedef struct I3DParams
{
    /* NLSSolver::setCostWeight(0..3): lambda_g, lambda_r(itr), lambda_s(itr), lambda_a */
    double lambda[I3D_NUM_COST_TYPES];
    /* term switches: E_r iff lambda_r0>0 && lambda_r1>0, E_s likewise, E_a iff lambda_a>0
     * (optimizer.cpp:239,249,259) */
    int32_t use_er, use_es, use_ea;
    /* lambda_a < 0  =>  every albedo is constant (optimizer.cpp:330-334) */
    int32_t fix_all_albedo;
    /* Optimizer::Data::thres_shell */
    double thres_shell;
    /* SDFColorization::Config::max_occlusion_distance (0 => no occlusion test), float like the reference */
    float occlusion_distance;
    /* SDFColorization::Config::max_num_observations (K); 0 => keep all frames */
    int32_t num_observations;
    /* Optimizer::Config::lm_steps  -> ceres max_num_iterations */
    int32_t lm_steps;
    int32_t fix_poses, fix_intrinsics, fix_distortion;

    /* ---- Ceres 2.1.0 defaults (restated; see oracle/oracle.cpp header) ---- */
    double initial_trust_region_radius;   /* 1e4  */
    double max_trust_region_radius;       /* 1e16 */
    double min_trust_region_radius;       /* 1e-32 */
    double min_relative_decrease;         /* 1e-3 */
    double min_lm_diagonal;               /* 1e-6 */
    double max_lm_diagonal;               /* 1e32 */
    double eta;                           /* 0.1  (CG q-tolerance) */
    double function_tolerance;            /* 1e-6 */
    double gradient_tolerance;            /* 1e-10 */
    double parameter_tolerance;           /* 1e-8 */
    int32_t max_linear_solver_iterations; /* 500 */
    int32_t min_linear_solver_iterations; /* 0 */
    int32_t residual_reset_period;        /* 10 */
    int32_t max_consecutive_invalid_steps;/* 5 */

    /* ---- test hooks (not in the reference) ---- */
    /* >0: every CGNR solve runs exactly this many iterations (parity tests compare
     * engine and oracle at an identical iteration count). */
    int32_t forced_cg_iterations;
    /* 1: evaluate and build the problem, but do not run the LM solve */
    int32_t build_only;
} I3DParams;

/* Mirrors NLSSolver::ProblemInfo + SolverInfo (L/include/nv/refinement/nls_solver.h:58-89)
 * plus what the parity tests need. */
typedef struct I3DIterInfo
{
    int64_t num_voxels;
    int64_t num_active;                       /* voxels passing addVoxelResiduals' tests */
    int64_t num_free_sdf, num_free_albedo;    /* by mask (fixVoxelParams) */
    int64_t num_parameters;                   /* free scalars incl. camera */
    int64_t type_residuals[I3D_NUM_COST_TYPES];
    double  type_sum_weights[I3D_NUM_COST_TYPES];  /* sum of raw residual weights per type */
    double  type_weights[I3D_NUM_COST_TYPES];      /* lambda/sum*1000 (ProblemInfo::type_weights) */
    double  type_costs[I3D_NUM_COST_TYPES];        /* 0.5*sum w r^2 at the initial point, per type */
    double  cost_initial;                     /* SolverInfo::cost        */
    double  cost_final;                       /* SolverInfo::cost_final  */
    double  trust_region_radius;              /* radius after the last LM iteration */
    int32_t lm_iterations;                    /* trial steps taken (SolverInfo::inner_iterations - 1) */
    int32_t step_accepted;                    /* 1 if a successful step was applied */
    int32_t termination;                      /* 0 user_success(first accepted step) 1 convergence
                                                 2 no_convergence 3 failure 4 nothing to do */
    int32_t cg_iterations_total;
    int32_t cg_iterations[I3D_MAX_LM_STEPS];  /* per trial */
    double  model_cost_change[I3D_MAX_LM_STEPS];
    double  candidate_cost[I3D_MAX_LM_STEPS];
    double  relative_decrease[I3D_MAX_LM_STEPS];
    double  step_norm;                        /* ||delta|| of the last evaluated trial (unscaled) */
    double  time_add, time_build, time_solve; /* seconds; the reference's three phase timers */
} I3DIterInfo;

/* ---- SVSH lighting (LightingSVSH, libintrinsic3d/src/lighting/lighting_svsh.cpp:54-346) ---- */
#define I3D_SH_COEFFS 9

/* Constructor arguments of LightingSVSH (include/nv/lighting/lighting_svsh.h:50) plus the Ceres
 * options LightingSVSH::estimate sets (lighting_svsh.cpp:186,325-337) and the Ceres 2.1.0
 * defaults it inherits. */
typedef struct I3DLightingParams
{
    float   subvolume_size;               /* Intrinsic3D::Config::subvolume_size_sh (0.2 m) */
    int32_t weighted;                     /* refine() passes true: weight = sdfToWeight(sdf_refined, truncation) */
    double  lambda_reg;                   /* sh_est_lambda_reg (10.0) */
    double  thres_shell;                  /* Optimizer::Data::thres_shell */
    int32_t max_iterations;               /* 50 (lighting_svsh.cpp:186) */
    int32_t max_linear_solver_iterations; /* 500 */
    int32_t min_linear_solver_iterations; /* 0 */
    int32_t residual_reset_period;        /* 10 */
    int32_t max_consecutive_invalid_steps;/* 5 */
    int32_t reserved;
    double  initial_trust_region_radius;  /* 1e4 */
    double  max_trust_region_radius;      /* 1e16 */
    double  min_trust_region_radius;      /* 1e-32 */
    double  min_relative_decrease;        /* 1e-3 */
    double  min_lm_diagonal;              /* 1e-6 */
    double  max_lm_diagonal;              /* 1e32 */
    double  eta;                          /* 0.1 */
    double  function_tolerance;           /* 1e-6 */
    double  gradient_tolerance;           /* 1e-10 */
    double  parameter_tolerance;          /* 1e-8 */
} I3DLightingParams;

/* What ceres::Solver::Summary would report for the SH problem, plus problem sizes. */
typedef struct I3DLightingInfo
{
    int64_t num_subvolumes;               /* Subvolumes::count() */
    int64_t num_data_rows;                /* SHDataCost residuals (one per contributing voxel) */
    int64_t num_reg_pairs;                /* SHRegularizerCost blocks (directed pairs, 9 residuals each) */
    double  sum_data_weights;
    double  cost_initial, cost_final;
    double  trust_region_radius;
    int32_t lm_iterations;                /* trust-region iterations started (Summary::iterations.size() - 1) */
    int32_t num_successful_steps;
    int32_t cg_iterations_total;
    int32_t termination;                  /* 0 convergence, 1 no_convergence (max iterations), 2 failure */
    int32_t usable;                       /* Summary::IsSolutionUsable() == the return value of estimate() */
    int32_t reserved;
    double  time_accumulate, time_solve, time_interpolate;   /* seconds (device time) */
} I3DLightingInfo;

/* ---- RGB-D fusion (AppFusion::fuseSDF, apps/src/app_fusion.cpp:107-200) ---- */
/* SparseVoxelGrid<Voxel>::create(voxel_size, depth_min, depth_max) (src/sparse_voxel_grid.cpp:42-64) plus the fusion config
 * (data/fusion.yml).  Truncation is 5 * voxel_size, as the reference's constructor sets it. */
typedef struct I3DFusionParams
{
    float   voxel_size;                   /* metres (fusion.yml: 0.004); must be > 1e-5 */
    float   depth_min, depth_max;         /* Sensor::depthMin / depthMax: frustum bounds and the depth weight */
    float   integration_weight_sample;    /* 10, the constant of SparseVoxelGrid's constructor; 0 = unit weights */
    float   clip_bounds[6];               /* x0,x1,y0,y1,z0,z1 in metres; all zero = off (the reference's norm() > 0 test) */
    int32_t discont_window_size;          /* erodeDiscontinuities window (fusion.yml: 2); 0 = no erosion */
    int32_t correct_sdf_iterations;       /* correctSDF sweeps at most (10) */
    int64_t initial_capacity;             /* hash slots to start with, 0 = default.  Only useful to force table growth in tests */
} I3DFusionParams;

/* A pinhole camera as Camera::project2 / unproject2 use it (src/camera.cpp:157-199): no distortion. */
typedef struct I3DFusionCamera
{
    int32_t width, height;
    float   fx, fy, cx, cy;
} I3DFusionCamera;

/* ---- surface extraction (MarchingCubes::extractSurface + MeshUtil, src/mesh/marching_cubes.cpp, src/mesh/util.cpp) ---- */
typedef struct I3DMeshParams
{
    int32_t sdf_source;                   /* 0 = sdf0 (what AppFusion meshes), 1 = sdf_refined (what onSDFRefined meshes) */
    int32_t largest_component_only;       /* 1 = MeshUtil::removeLooseComponents + removeUnusedVertices (output_mesh_largest_comp_only) */
} I3DMeshParams;

typedef struct I3DMeshInfo
{
    int64_t num_cubes;                    /* cubes whose 8 corners exist with weight != 0 */
    int64_t num_faces_raw;                /* triangles emitted by marching cubes */
    int64_t num_vertices_welded;          /* distinct float positions among their corners */
    int64_t num_faces_clean;              /* faces left by removeDegenerateFaces */
    int64_t num_faces, num_vertices;      /* the resident mesh: after the component filter when asked for, else the cleaned faces and
                                             every welded vertex */
    double  ms_classify, ms_emit, ms_weld, ms_clean, ms_components;   /* device time per stage: CUDA events around its device-only
                                                                           segments, the host read-backs of counts excluded */
} I3DMeshInfo;

/* ---- simplifying the resident mesh: quadric-error vertex clustering (Lindstrom 2000; DESIGN.md §6s) ---- */
typedef struct I3DSimplifyParams
{
    float   cell_size;                    /* edge of the world-aligned cubic cells, metres (> 0, finite) */
    int32_t reserved;
} I3DSimplifyParams;

typedef struct I3DSimplifyInfo
{
    int64_t num_clusters;                 /* occupied cells = vertices before the unused ones are removed */
    int64_t num_faces_collapsed;          /* faces whose three corners fall into fewer than three clusters */
    int64_t num_faces_duplicate;          /* faces that repeat an earlier face up to rotation */
    int64_t num_faces_degenerate;         /* faces left that the extraction's degenerate-face rule drops at the representatives */
    int64_t num_faces, num_vertices;      /* the new resident mesh */
    double  ms_cluster, ms_quadrics, ms_representatives, ms_faces, ms_compact;   /* device time per stage: CUDA events around its
                                                                                     device-only segments, as in I3DMeshInfo */
} I3DSimplifyInfo;

/* ---- baking the keyframes' colour into a texture atlas of the resident mesh (DESIGN.md §6t) ---- */
#define I3D_TEXTURE_MIN_TEXELS_PER_FACE 6
#define I3D_TEXTURE_MAX_TEXELS_PER_FACE 256
#define I3D_TEXTURE_MAX_SIDE 16384      /* largest atlas width or height, texels */

typedef struct I3DTextureParams
{
    int32_t texels_per_face;              /* S: faces 2c and 2c+1 share cell c of S x S texels; in [6, 256] */
    float   max_occlusion_distance;       /* as i3d_recompute_colors: |depth - z| bound of an observation, metres; <= 0 turns the test off */
    int32_t max_num_observations;         /* K in [0, I3D_MAX_OBS]: the best K frames per texel; 0 = every observation */
    int32_t reserved;
} I3DTextureParams;

typedef struct I3DTextureInfo
{
    int32_t atlas_width, atlas_height;    /* texels */
    int64_t num_faces;                    /* faces of the resident mesh = UV triangles */
    int64_t num_texels_owned;             /* texels some face owns: num_faces * S (S - 1) / 2 */
    int64_t num_texels_observed;          /* owned texels with at least one observation: coloured from the keyframes */
    int64_t num_texels_fallback;          /* owned texels without one: the barycentric blend of the face's vertex colours */
    int64_t num_observations;             /* (texel, frame) pairs with weight > 0 */
    int64_t num_observations_kept;        /* observations summed into a colour: min(observations, K) per texel (all of them for K = 0) */
    int64_t num_texel_frames_visited;     /* (owned texel, frame) pairs whose weight was computed: the ones the frame culling kept */
    int64_t num_texel_frames_total;       /* owned texels x frames */
    double  ms_bake;                      /* device time of the bake and the UVs (CUDA events) */
} I3DTextureInfo;

/* ---- albedo and shading of the baked texture, and relighting (DESIGN.md §6x) ---- */
/* Lighting sources (I3DShLighting::source) */
enum { I3D_SH_ESTIMATE = 0, I3D_SH_GLOBAL = 1 };

/* A second-order SH lighting: the subvolume SH of the last i3d_estimate_lighting (blended at each point as the shading colour modes
 * blend it), or the same nine coefficients everywhere */
typedef struct I3DShLighting
{
    int32_t source;                       /* I3D_SH_* */
    int32_t reserved;
    float   sh[9];                        /* I3D_SH_GLOBAL: the coefficients, in the order of the lighting estimate; ignored otherwise */
} I3DShLighting;

typedef struct I3DIntrinsicTextureParams
{
    I3DShLighting lighting;
    float   min_shading;                  /* a texel is lit iff its face normal is not 0 and its shading s > min_shading (finite, >= 0) */
    int32_t reserved;
} I3DIntrinsicTextureParams;

typedef struct I3DIntrinsicTextureInfo
{
    int32_t atlas_width, atlas_height;    /* texels, as the texture's */
    int64_t num_texels_owned;             /* texels some face owns */
    int64_t num_texels_lit;               /* owned texels with a non-zero face normal and s > min_shading: albedo = colour / 255 / s */
    int64_t num_texels_unlit;             /* the other owned texels: albedo 0 */
    int64_t num_texels_lit_fallback;      /* lit texels the bake coloured from the vertex colours (no keyframe observed them) */
    float   albedo_min[3], albedo_max[3]; /* per channel R, G, B over the lit texels (0 without one) */
    double  ms_decompose;                 /* device time (CUDA events) */
} I3DIntrinsicTextureInfo;

/* ---- distance from the resident mesh to a reference mesh (DESIGN.md §6u) ---- */
#define I3D_DISTANCE_MAX_THRESHOLDS 8
#define I3D_DISTANCE_MAX_SAMPLES_PER_EDGE 16
#define I3D_DISTANCE_MAX_CELLS (1ll << 26)           /* largest search grid, cells */
#define I3D_DISTANCE_MAX_CELL_ENTRIES (1ll << 30)    /* largest (face, cell) list of a search grid */

typedef struct I3DDistanceParams
{
    int32_t samples_per_edge;             /* L in [1, 16]: every face is split into L^2 congruent sub-triangles, sampled at their centroids */
    float   max_distance;                 /* metres, finite and > 0: a sample with no face within it is unmatched */
    float   cell_size;                    /* search-grid cell edge, metres; 0 = twice the target mesh's mean edge length */
    int32_t num_thresholds;               /* in [0, 8] */
    float   thresholds[I3D_DISTANCE_MAX_THRESHOLDS];  /* tau: finite, ascending, <= max_distance */
} I3DDistanceParams;

/* One direction: the samples of one mesh against the faces of the other (the target) */
typedef struct I3DDistanceSide
{
    int64_t num_samples, num_matched;
    double  area;                         /* total sample weight = the sampled mesh's area, m^2 */
    double  unmatched_area;
    double  mean, rms, max;               /* of d over the matched samples, area-weighted (max: one-sided Hausdorff within max_distance) */
    double  fraction[I3D_DISTANCE_MAX_THRESHOLDS];   /* area with d <= tau over the total area; unmatched samples count as beyond every tau */
    int64_t point_triangle_tests;         /* closest-point evaluations of the query */
    float   cell_size;                    /* the target's search grid: cell edge (metres) and cells per axis */
    int32_t grid[3];
    int64_t num_cells, num_cell_entries;  /* cells, (face, cell) pairs */
    double  ms_grid, ms_query, ms_reduce; /* device time: grid build, sampling and query, statistics (CUDA events) */
} I3DDistanceSide;

typedef struct I3DDistanceInfo
{
    I3DDistanceSide side[2];              /* [0] resident -> reference (accuracy, precision), [1] reference -> resident (completeness, recall) */
    int32_t num_thresholds, reserved;
    double  precision[I3D_DISTANCE_MAX_THRESHOLDS], recall[I3D_DISTANCE_MAX_THRESHOLDS], fscore[I3D_DISTANCE_MAX_THRESHOLDS];
    int64_t num_vertices;                 /* vertices of the resident mesh, each queried against the reference */
    int64_t vertex_point_triangle_tests;
    double  ms_vertices;                  /* device time of the vertex query */
} I3DDistanceInfo;

/* ---- the voxel grid from a triangle mesh: narrow-band signed distance (DESIGN.md §6v) ---- */
#define I3D_GRID_FROM_MESH_REFERENCE 0      /* source: the mesh of i3d_upload_reference_mesh */
#define I3D_GRID_FROM_MESH_RESIDENT 1       /* source: the resident mesh (the last extraction or simplification) */
#define I3D_GRID_FROM_MESH_MAX_BAND 16.0f   /* largest band, voxels */
#define I3D_GRID_FROM_MESH_MAX_PAIRS (1ll << 28)     /* largest sum over faces of the 8^3 bricks their band-grown AABB covers */
#define I3D_GRID_FROM_MESH_MAX_VOXELS (1ll << 30)    /* largest number of candidate voxels (512 per candidate brick) */
/* A voxel whose closest feature is a boundary edge or vertex is kept only when |cos| of the angle between p - q and the feature's
 * pseudonormal is >= this: an open mesh grows no skirt past its rim */
#define I3D_GRID_FROM_MESH_RIM_COS 0.5

typedef struct I3DGridFromMeshParams
{
    int32_t source;                       /* I3D_GRID_FROM_MESH_REFERENCE or I3D_GRID_FROM_MESH_RESIDENT */
    float   voxel_size;                   /* metres, finite and > 0: voxel c sits at c * voxel_size */
    float   band;                         /* voxels, in (0, 16]: voxels with a face within band * voxel_size are emitted */
    float   cell_size;                    /* search-grid cell edge, metres; 0 = twice the mesh's mean edge length.  Never changes the result */
} I3DGridFromMeshParams;

typedef struct I3DGridFromMeshInfo
{
    int64_t num_faces;                    /* faces of the source mesh */
    int64_t num_vertices_welded;          /* distinct vertex positions */
    int64_t num_boundary_edges;           /* welded edges used by exactly one non-degenerate face */
    int64_t num_brick_pairs;              /* (face, brick) pairs of the band-grown face AABBs, before the distance test */
    int64_t num_candidate_bricks, num_candidate_voxels;
    int64_t num_voxels, num_negative;     /* emitted voxels, and those with sdf < 0 */
    int64_t num_beyond_band;              /* candidate voxels with no face within the band */
    int64_t num_dropped_rim;              /* closest feature on the boundary and |cos| < I3D_GRID_FROM_MESH_RIM_COS */
    int64_t num_dropped_zero_normal;      /* closest feature with a zero pseudonormal */
    int64_t num_dropped_zero_dot;         /* d > 0 and p - q orthogonal to the pseudonormal: no sign */
    int64_t point_triangle_tests;         /* closest-point evaluations of the query */
    float   cell_size;                    /* the search grid used: cell edge (metres) and cells per axis */
    int32_t grid[3];
    double  ms_topology, ms_grid, ms_bricks, ms_query, ms_install;   /* device time per stage (CUDA events) */
} I3DGridFromMeshInfo;

/* Features of the closest point on a face (i3d_debug_get_grid_from_mesh_voxels): vertex a, b, c, edge ab, ac, bc, interior */
enum { I3D_FEATURE_VERTEX_A = 0, I3D_FEATURE_VERTEX_B, I3D_FEATURE_VERTEX_C, I3D_FEATURE_EDGE_AB, I3D_FEATURE_EDGE_AC, I3D_FEATURE_EDGE_BC,
       I3D_FEATURE_INTERIOR };

/* Colour modes of a mesh (SDFVisualization::colorize, src/sdf/visualization.cpp:101-416; mode strings "", "normals", "lap", "lum",
 * "lum_grad", "albedo", "shading_sv", "shading_sv_const", "chroma").  VOXEL is the voxel colours; the others are computed per voxel from
 * the voxel and its ±1 ring (DESIGN.md §6k).  The reference's subvolume modes ("subvol", "subvol_interp") have no number. */
enum
{
    I3D_MESH_COLOR_VOXEL = 0,
    I3D_MESH_COLOR_NORMALS,
    I3D_MESH_COLOR_LAPLACIAN,
    I3D_MESH_COLOR_INTENSITY,
    I3D_MESH_COLOR_INTENSITY_GRAD,
    I3D_MESH_COLOR_ALBEDO,
    I3D_MESH_COLOR_SHADING_SV,
    I3D_MESH_COLOR_SHADING_SV_CONST,
    I3D_MESH_COLOR_CHROMACITY,
    I3D_MESH_COLOR_COUNT
};

/* ---- rendering the surface into the keyframes (DESIGN.md §6m) ---- */
/* Planes of a render (bit mask of I3DRenderParams::planes). */
enum
{
    I3D_RENDER_DEPTH = 1,                 /* camera z of the hit, 0 = no hit */
    I3D_RENDER_NORMAL = 2,                /* unit sdf gradient at the hit, world frame, [3] per pixel; (0,0,0) = none */
    I3D_RENDER_ALBEDO = 4,                /* trilinear albedo at the hit */
    I3D_RENDER_SHADING = 8,               /* shading(normal, per-voxel SH) at the hit, 0 where undefined */
    I3D_RENDER_INTENSITY = 16,            /* albedo * shading, 0 where undefined */
    I3D_RENDER_ALL = 31
};

typedef struct I3DRenderParams
{
    int32_t sdf_source;                   /* 0 = sdf0, 1 = sdf_refined, as in I3DMeshParams */
    int32_t planes;                       /* I3D_RENDER_* mask; 0 = statistics only (no plane buffers) */
    int32_t photometric;                  /* 1 = photometric pairs (needs the per-voxel SH); 0 = geometry only */
    int32_t reserved;
} I3DRenderParams;

/* Per-view comparison of a render with its keyframe.  Sums are double, in a fixed order: a view's numbers depend only on that view. */
typedef struct I3DRenderStats
{
    int64_t num_hit;                      /* pixels whose ray hit the surface */
    int64_t num_observed;                 /* pixels with input depth > 0 */
    int64_t depth_count;                  /* hit and observed */
    int64_t photo_count;                  /* hit, shading defined and observed (0 when photometric = 0) */
    double  depth_abs, depth_sq;          /* sum |z_r - z_obs|, sum (z_r - z_obs)^2 over the depth pairs (metres) */
    double  photo_abs, photo_sq;          /* sum |I_r - I_obs|, sum (I_r - I_obs)^2 over the photometric pairs (I_obs: the frame's luminance) */
} I3DRenderStats;

/* ---- rasterizing the resident mesh into the keyframes and into new views (DESIGN.md §6w) ---- */
/* Planes of a rasterization (bit mask of I3DRasterParams::planes). */
enum
{
    I3D_RASTER_DEPTH = 1,                 /* float camera z of the nearest face, 0 = no hit */
    I3D_RASTER_FACE = 2,                  /* int32 face id, -1 = no hit */
    I3D_RASTER_BARY = 4,                  /* float [2]: barycentric weights (a, b) of v1, v2; w0 = (1 - a) - b; 0 = no hit */
    I3D_RASTER_NORMAL = 8,                /* float [3]: unit face normal, world frame; (0,0,0) = no hit or zero area */
    I3D_RASTER_RGB = 16,                  /* uint8 [3]: R, G, B of the colour source; 0 = no hit or no source */
    I3D_RASTER_ALL = 31
};
/* Colour sources (I3DRasterParams::color_source) */
enum { I3D_RASTER_COLOR_NONE = 0, I3D_RASTER_COLOR_VERTEX = 1, I3D_RASTER_COLOR_TEXTURE = 2,
       I3D_RASTER_COLOR_RELIT = 3 /* albedo of i3d_decompose_texture x shading under the lighting of i3d_set_relight */ };
#define I3D_RASTER_MAX_SIDE 8192          /* largest width or height of a new view */

typedef struct I3DRasterParams
{
    int32_t planes;                       /* I3D_RASTER_* mask; 0 = statistics only (no plane buffers) */
    int32_t color_source;                 /* I3D_RASTER_COLOR_* */
    int32_t reserved[2];
} I3DRasterParams;

/* A camera of new views: intrinsics in pixels of a width x height image, and the five distortion coefficients (k1, k2, p1, p2, k3) */
typedef struct I3DRasterCamera
{
    float   fx, fy, cx, cy;
    float   distortion[5];
    int32_t width, height;
} I3DRasterCamera;

/* Per-keyframe comparison of the rasterized mesh with the keyframe's depth and colour.  Depth sums are double in a fixed order, colour
 * sums exact integers: a view's numbers depend only on that view. */
typedef struct I3DRasterStats
{
    int64_t num_covered;                  /* pixels some face covers */
    int64_t num_observed;                 /* pixels with frame depth > 0 */
    int64_t depth_count;                  /* covered and observed */
    int64_t color_count;                  /* covered, with a colour source (0 without one) */
    double  depth_abs, depth_sq;          /* sum |e|, sum e^2 over the depth pairs, e = double(z_mesh) - double(z_frame), metres */
    int64_t color_abs[3], color_sq[3];    /* per channel R, G, B: sum |e|, sum e^2 over the colour pairs, e = rendered - frame (uint8 units) */
} I3DRasterStats;

typedef struct I3DRasterInfo
{
    int64_t num_views, num_faces;         /* views of the call, faces of the resident mesh */
    int64_t num_pairs;                    /* (8 x 8 tile, face) pairs the binning kept, over all views */
    int64_t num_straddling;               /* (face, view) pairs with camera z <= 0 and > 0 among the vertices: binned to every tile */
    int64_t num_behind;                   /* (face, view) pairs with every camera z <= 0: never hit, dropped */
    int64_t num_tests;                    /* ray-triangle tests */
    int64_t num_covered;                  /* covered pixels over all views */
    double  ms_rays, ms_faces, ms_shade;  /* device time: ray table and tile boxes, face binning and tests, shading and statistics */
} I3DRasterInfo;

/* ---- tracking sensor frames against the surface: point-to-plane ICP over the depth pyramid (DESIGN.md §6n) ---- */
/* Per-frame outcome of a tracking call (I3DTrackInfo::status). */
enum
{
    I3D_TRACK_OK = 0,                     /* every scheduled update applied */
    I3D_TRACK_FEW_CORRESPONDENCES = 1,    /* a system had fewer than min_correspondences rows: frozen there */
    I3D_TRACK_NOT_POSITIVE_DEFINITE = 2,  /* the Cholesky factorisation of a system failed: frozen there */
    I3D_TRACK_NON_FINITE = 3,             /* a system, its update or the updated pose was not finite: frozen there */
    I3D_TRACK_ANCHORED = 4                /* odometry: the volume had no integrated voxel; the frame was integrated at its guess untracked */
};

typedef struct I3DTrackParams
{
    int32_t sdf_source;                   /* 0 = sdf0, 1 = sdf_refined, as in I3DMeshParams / I3DRenderParams */
    int32_t num_levels;                   /* depth pyramid levels, 1..4 */
    int32_t iterations[4];                /* Gauss-Newton iterations per level, level 0 first; the coarsest level runs first */
    float   max_distance;                 /* correspondence gate |p - q|, metres */
    float   min_normal_cos;               /* correspondence gate n_in . n_model; -1 = off */
    int32_t min_correspondences;          /* fewer rows at a solve freeze the frame (>= 6) */
    int32_t reserved;
} I3DTrackParams;

typedef struct I3DTrackInfo
{
    int32_t        status;                /* I3D_TRACK_* */
    int32_t        iterations;            /* updates applied before the frame froze or finished */
    int64_t        correspondences;       /* rows of the last evaluated system */
    double         residual_sq;           /* sum of squared point-to-plane residuals of that system (metres^2) */
    double         update_norm;           /* |xi| of the last applied update (0 without one) */
    I3DRenderStats initial;               /* the prediction render against the frame's depth, at the input pose */
} I3DTrackInfo;

/* ---- the photometric term of tracking: joint depth and colour Gauss-Newton (DESIGN.md §6p) ---- */
typedef struct I3DTrackColorParams
{
    float   weight[4];                    /* lambda per pyramid level, level 0 first: A = A_depth + lambda^2 A_colour; 0 = depth only */
    float   max_color_diff;               /* photometric gate |I_frame - I_model| (intensity in [0, 1]) */
    float   min_color_gradient;           /* texture gate |grad I_frame| (intensity per pixel, central differences); 0 = off */
    int32_t norm_radius;                  /* _ref calls only: > 0 compares locally normalised intensity over (2r+1)^2 windows (DESIGN.md
                                             section 6r), and max_color_diff and min_color_gradient are then in its units; 0 = raw intensity */
    float   norm_eps;                     /* with norm_radius > 0: the normalisation's floor, (I - mu) / sqrt(var + norm_eps^2); > 0 */
} I3DTrackColorParams;

typedef struct I3DTrackColorInfo
{
    int64_t first_rows;                   /* photometric rows of the first evaluated system (at the input pose, coarsest level) */
    double  first_residual_sq;            /* sum of their squared intensity residuals */
    int64_t last_rows;                    /* photometric rows of the last evaluated system */
    double  last_residual_sq;
} I3DTrackColorInfo;

#ifdef __cplusplus
}
#endif
#endif /* I3D_TYPES_H_ */
