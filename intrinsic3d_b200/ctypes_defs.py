"""ctypes mirrors of include/i3d_types.h (I3DParams / I3DIterInfo / I3DLightingParams / I3DLightingInfo).

Field order and types must match the C header exactly; tests/test_abi.py checks
sizeof() against the compiled library.
"""
import ctypes as C

NUM_COST_TYPES = 4
MAX_OBS = 8
EG_COLS = 29
MAX_LM_STEPS = 64


class I3DParams(C.Structure):
    _fields_ = [
        ("lambda_", C.c_double * NUM_COST_TYPES),
        ("use_er", C.c_int32),
        ("use_es", C.c_int32),
        ("use_ea", C.c_int32),
        ("fix_all_albedo", C.c_int32),
        ("thres_shell", C.c_double),
        ("occlusion_distance", C.c_float),
        ("num_observations", C.c_int32),
        ("lm_steps", C.c_int32),
        ("fix_poses", C.c_int32),
        ("fix_intrinsics", C.c_int32),
        ("fix_distortion", C.c_int32),
        ("initial_trust_region_radius", C.c_double),
        ("max_trust_region_radius", C.c_double),
        ("min_trust_region_radius", C.c_double),
        ("min_relative_decrease", C.c_double),
        ("min_lm_diagonal", C.c_double),
        ("max_lm_diagonal", C.c_double),
        ("eta", C.c_double),
        ("function_tolerance", C.c_double),
        ("gradient_tolerance", C.c_double),
        ("parameter_tolerance", C.c_double),
        ("max_linear_solver_iterations", C.c_int32),
        ("min_linear_solver_iterations", C.c_int32),
        ("residual_reset_period", C.c_int32),
        ("max_consecutive_invalid_steps", C.c_int32),
        ("forced_cg_iterations", C.c_int32),
        ("build_only", C.c_int32),
    ]


class I3DIterInfo(C.Structure):
    _fields_ = [
        ("num_voxels", C.c_int64),
        ("num_active", C.c_int64),
        ("num_free_sdf", C.c_int64),
        ("num_free_albedo", C.c_int64),
        ("num_parameters", C.c_int64),
        ("type_residuals", C.c_int64 * NUM_COST_TYPES),
        ("type_sum_weights", C.c_double * NUM_COST_TYPES),
        ("type_weights", C.c_double * NUM_COST_TYPES),
        ("type_costs", C.c_double * NUM_COST_TYPES),
        ("cost_initial", C.c_double),
        ("cost_final", C.c_double),
        ("trust_region_radius", C.c_double),
        ("lm_iterations", C.c_int32),
        ("step_accepted", C.c_int32),
        ("termination", C.c_int32),
        ("cg_iterations_total", C.c_int32),
        ("cg_iterations", C.c_int32 * MAX_LM_STEPS),
        ("model_cost_change", C.c_double * MAX_LM_STEPS),
        ("candidate_cost", C.c_double * MAX_LM_STEPS),
        ("relative_decrease", C.c_double * MAX_LM_STEPS),
        ("step_norm", C.c_double),
        ("time_add", C.c_double),
        ("time_build", C.c_double),
        ("time_solve", C.c_double),
    ]

    def as_dict(self):
        out = {}
        for name, _ in self._fields_:
            v = getattr(self, name)
            out[name] = list(v) if hasattr(v, "__len__") else v
        return out


def default_params() -> I3DParams:
    """Defaults = data/intrinsic3d.yml (first outer iteration) + Ceres 2.1.0 solver defaults."""
    p = I3DParams()
    p.lambda_[0], p.lambda_[1], p.lambda_[2], p.lambda_[3] = 0.2, 80.0, 120.0, 0.1
    p.use_er = p.use_es = p.use_ea = 1
    p.fix_all_albedo = 0
    p.thres_shell = 0.0
    p.occlusion_distance = 0.02
    p.num_observations = 5
    p.lm_steps = 50
    p.initial_trust_region_radius = 1e4
    p.max_trust_region_radius = 1e16
    p.min_trust_region_radius = 1e-32
    p.min_relative_decrease = 1e-3
    p.min_lm_diagonal = 1e-6
    p.max_lm_diagonal = 1e32
    p.eta = 0.1
    p.function_tolerance = 1e-6
    p.gradient_tolerance = 1e-10
    p.parameter_tolerance = 1e-8
    p.max_linear_solver_iterations = 500
    p.min_linear_solver_iterations = 0
    p.residual_reset_period = 10
    p.max_consecutive_invalid_steps = 5
    return p


class _Dictable:
    def as_dict(self):
        out = {}
        for name, _ in self._fields_:
            v = getattr(self, name)
            out[name] = list(v) if hasattr(v, "__len__") else v
        return out


class I3DLightingParams(C.Structure, _Dictable):
    _fields_ = [
        ("subvolume_size", C.c_float),
        ("weighted", C.c_int32),
        ("lambda_reg", C.c_double),
        ("thres_shell", C.c_double),
        ("max_iterations", C.c_int32),
        ("max_linear_solver_iterations", C.c_int32),
        ("min_linear_solver_iterations", C.c_int32),
        ("residual_reset_period", C.c_int32),
        ("max_consecutive_invalid_steps", C.c_int32),
        ("reserved", C.c_int32),
        ("initial_trust_region_radius", C.c_double),
        ("max_trust_region_radius", C.c_double),
        ("min_trust_region_radius", C.c_double),
        ("min_relative_decrease", C.c_double),
        ("min_lm_diagonal", C.c_double),
        ("max_lm_diagonal", C.c_double),
        ("eta", C.c_double),
        ("function_tolerance", C.c_double),
        ("gradient_tolerance", C.c_double),
        ("parameter_tolerance", C.c_double),
    ]


class I3DLightingInfo(C.Structure, _Dictable):
    _fields_ = [
        ("num_subvolumes", C.c_int64),
        ("num_data_rows", C.c_int64),
        ("num_reg_pairs", C.c_int64),
        ("sum_data_weights", C.c_double),
        ("cost_initial", C.c_double),
        ("cost_final", C.c_double),
        ("trust_region_radius", C.c_double),
        ("lm_iterations", C.c_int32),
        ("num_successful_steps", C.c_int32),
        ("cg_iterations_total", C.c_int32),
        ("termination", C.c_int32),
        ("usable", C.c_int32),
        ("reserved", C.c_int32),
        ("time_accumulate", C.c_double),
        ("time_solve", C.c_double),
        ("time_interpolate", C.c_double),
    ]


class I3DFusionParams(C.Structure, _Dictable):
    _fields_ = [
        ("voxel_size", C.c_float),
        ("depth_min", C.c_float),
        ("depth_max", C.c_float),
        ("integration_weight_sample", C.c_float),
        ("clip_bounds", C.c_float * 6),
        ("discont_window_size", C.c_int32),
        ("correct_sdf_iterations", C.c_int32),
        ("initial_capacity", C.c_int64),
    ]


class I3DFusionCamera(C.Structure, _Dictable):
    _fields_ = [
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("fx", C.c_float),
        ("fy", C.c_float),
        ("cx", C.c_float),
        ("cy", C.c_float),
    ]


class I3DMeshParams(C.Structure, _Dictable):
    _fields_ = [
        ("sdf_source", C.c_int32),
        ("largest_component_only", C.c_int32),
    ]


class I3DMeshInfo(C.Structure, _Dictable):
    _fields_ = [
        ("num_cubes", C.c_int64),
        ("num_faces_raw", C.c_int64),
        ("num_vertices_welded", C.c_int64),
        ("num_faces_clean", C.c_int64),
        ("num_faces", C.c_int64),
        ("num_vertices", C.c_int64),
        ("ms_classify", C.c_double),
        ("ms_emit", C.c_double),
        ("ms_weld", C.c_double),
        ("ms_clean", C.c_double),
        ("ms_components", C.c_double),
    ]


class I3DSimplifyParams(C.Structure, _Dictable):
    _fields_ = [
        ("cell_size", C.c_float),
        ("reserved", C.c_int32),
    ]


class I3DSimplifyInfo(C.Structure, _Dictable):
    _fields_ = [
        ("num_clusters", C.c_int64),
        ("num_faces_collapsed", C.c_int64),
        ("num_faces_duplicate", C.c_int64),
        ("num_faces_degenerate", C.c_int64),
        ("num_faces", C.c_int64),
        ("num_vertices", C.c_int64),
        ("ms_cluster", C.c_double),
        ("ms_quadrics", C.c_double),
        ("ms_representatives", C.c_double),
        ("ms_faces", C.c_double),
        ("ms_compact", C.c_double),
    ]


class I3DTextureParams(C.Structure, _Dictable):
    _fields_ = [
        ("texels_per_face", C.c_int32),
        ("max_occlusion_distance", C.c_float),
        ("max_num_observations", C.c_int32),
        ("reserved", C.c_int32),
    ]


class I3DTextureInfo(C.Structure, _Dictable):
    _fields_ = [
        ("atlas_width", C.c_int32),
        ("atlas_height", C.c_int32),
        ("num_faces", C.c_int64),
        ("num_texels_owned", C.c_int64),
        ("num_texels_observed", C.c_int64),
        ("num_texels_fallback", C.c_int64),
        ("num_observations", C.c_int64),
        ("num_observations_kept", C.c_int64),
        ("num_texel_frames_visited", C.c_int64),
        ("num_texel_frames_total", C.c_int64),
        ("ms_bake", C.c_double),
    ]


SH_SOURCES = {"estimate": 0, "global": 1}     # I3D_SH_* of include/i3d_types.h


class I3DShLighting(C.Structure, _Dictable):
    _fields_ = [
        ("source", C.c_int32),
        ("reserved", C.c_int32),
        ("sh", C.c_float * 9),
    ]


class I3DIntrinsicTextureParams(C.Structure, _Dictable):
    _fields_ = [
        ("lighting", I3DShLighting),
        ("min_shading", C.c_float),
        ("reserved", C.c_int32),
    ]


class I3DIntrinsicTextureInfo(C.Structure, _Dictable):
    _fields_ = [
        ("atlas_width", C.c_int32),
        ("atlas_height", C.c_int32),
        ("num_texels_owned", C.c_int64),
        ("num_texels_lit", C.c_int64),
        ("num_texels_unlit", C.c_int64),
        ("num_texels_lit_fallback", C.c_int64),
        ("albedo_min", C.c_float * 3),
        ("albedo_max", C.c_float * 3),
        ("ms_decompose", C.c_double),
    ]


DISTANCE_MAX_THRESHOLDS = 8     # I3D_DISTANCE_MAX_THRESHOLDS of include/i3d_types.h


class I3DDistanceParams(C.Structure, _Dictable):
    _fields_ = [
        ("samples_per_edge", C.c_int32),
        ("max_distance", C.c_float),
        ("cell_size", C.c_float),
        ("num_thresholds", C.c_int32),
        ("thresholds", C.c_float * DISTANCE_MAX_THRESHOLDS),
    ]


class I3DDistanceSide(C.Structure, _Dictable):
    _fields_ = [
        ("num_samples", C.c_int64),
        ("num_matched", C.c_int64),
        ("area", C.c_double),
        ("unmatched_area", C.c_double),
        ("mean", C.c_double),
        ("rms", C.c_double),
        ("max", C.c_double),
        ("fraction", C.c_double * DISTANCE_MAX_THRESHOLDS),
        ("point_triangle_tests", C.c_int64),
        ("cell_size", C.c_float),
        ("grid", C.c_int32 * 3),
        ("num_cells", C.c_int64),
        ("num_cell_entries", C.c_int64),
        ("ms_grid", C.c_double),
        ("ms_query", C.c_double),
        ("ms_reduce", C.c_double),
    ]


class I3DDistanceInfo(C.Structure, _Dictable):
    _fields_ = [
        ("side", I3DDistanceSide * 2),
        ("num_thresholds", C.c_int32),
        ("reserved", C.c_int32),
        ("precision", C.c_double * DISTANCE_MAX_THRESHOLDS),
        ("recall", C.c_double * DISTANCE_MAX_THRESHOLDS),
        ("fscore", C.c_double * DISTANCE_MAX_THRESHOLDS),
        ("num_vertices", C.c_int64),
        ("vertex_point_triangle_tests", C.c_int64),
        ("ms_vertices", C.c_double),
    ]


REGISTER_MAX_STAGES = 4          # I3D_REGISTER_MAX_STAGES of include/i3d_types.h


class I3DRegisterParams(C.Structure, _Dictable):
    _fields_ = [
        ("samples_per_edge", C.c_int32),
        ("num_stages", C.c_int32),
        ("max_distance", C.c_float * REGISTER_MAX_STAGES),
        ("iterations", C.c_int32 * REGISTER_MAX_STAGES),
        ("min_normal_cos", C.c_float),
        ("min_correspondences", C.c_int32),
        ("cell_size", C.c_float),
    ]


class I3DRegisterInfo(C.Structure, _Dictable):
    _fields_ = [
        ("status", C.c_int32),
        ("iterations", C.c_int32),
        ("initial_rows", C.c_int64),
        ("final_rows", C.c_int64),
        ("initial_weight", C.c_double),
        ("final_weight", C.c_double),
        ("initial_residual_sq", C.c_double),
        ("final_residual_sq", C.c_double),
        ("initial_rms", C.c_double),
        ("final_rms", C.c_double),
        ("update_norm", C.c_double),
        ("num_samples", C.c_int64),
        ("point_triangle_tests", C.c_int64),
        ("cell_size", C.c_float),
        ("grid", C.c_int32 * 3),
        ("num_cells", C.c_int64),
        ("num_cell_entries", C.c_int64),
        ("ms_grid", C.c_double),
        ("ms_rows", C.c_double),
        ("ms_solve", C.c_double),
    ]


# I3D_GRID_FROM_MESH_* sources of include/i3d_types.h
GRID_FROM_MESH_SOURCES = {"reference": 0, "resident": 1}


class I3DGridFromMeshParams(C.Structure, _Dictable):
    _fields_ = [
        ("source", C.c_int32),
        ("voxel_size", C.c_float),
        ("band", C.c_float),
        ("cell_size", C.c_float),
    ]


class I3DGridFromMeshInfo(C.Structure, _Dictable):
    _fields_ = [
        ("num_faces", C.c_int64),
        ("num_vertices_welded", C.c_int64),
        ("num_boundary_edges", C.c_int64),
        ("num_brick_pairs", C.c_int64),
        ("num_candidate_bricks", C.c_int64),
        ("num_candidate_voxels", C.c_int64),
        ("num_voxels", C.c_int64),
        ("num_negative", C.c_int64),
        ("num_beyond_band", C.c_int64),
        ("num_dropped_rim", C.c_int64),
        ("num_dropped_zero_normal", C.c_int64),
        ("num_dropped_zero_dot", C.c_int64),
        ("point_triangle_tests", C.c_int64),
        ("cell_size", C.c_float),
        ("grid", C.c_int32 * 3),
        ("ms_topology", C.c_double),
        ("ms_grid", C.c_double),
        ("ms_bricks", C.c_double),
        ("ms_query", C.c_double),
        ("ms_install", C.c_double),
    ]


# I3D_RENDER_* plane bits of include/i3d_types.h
RENDER_PLANES = {"depth": 1, "normal": 2, "albedo": 4, "shading": 8, "intensity": 16}


class I3DRenderParams(C.Structure, _Dictable):
    _fields_ = [
        ("sdf_source", C.c_int32),
        ("planes", C.c_int32),
        ("photometric", C.c_int32),
        ("reserved", C.c_int32),
    ]


class I3DRenderStats(C.Structure, _Dictable):
    _fields_ = [
        ("num_hit", C.c_int64),
        ("num_observed", C.c_int64),
        ("depth_count", C.c_int64),
        ("photo_count", C.c_int64),
        ("depth_abs", C.c_double),
        ("depth_sq", C.c_double),
        ("photo_abs", C.c_double),
        ("photo_sq", C.c_double),
    ]


# I3D_RASTER_* plane bits and colour sources of include/i3d_types.h
RASTER_PLANES = {"depth": 1, "face": 2, "bary": 4, "normal": 8, "rgb": 16}
RASTER_COLORS = {None: 0, "vertex": 1, "texture": 2, "relit": 3}


class I3DRasterParams(C.Structure, _Dictable):
    _fields_ = [
        ("planes", C.c_int32),
        ("color_source", C.c_int32),
        ("reserved", C.c_int32 * 2),
    ]


class I3DRasterCamera(C.Structure, _Dictable):
    _fields_ = [
        ("fx", C.c_float),
        ("fy", C.c_float),
        ("cx", C.c_float),
        ("cy", C.c_float),
        ("distortion", C.c_float * 5),
        ("width", C.c_int32),
        ("height", C.c_int32),
    ]


class I3DRasterStats(C.Structure, _Dictable):
    _fields_ = [
        ("num_covered", C.c_int64),
        ("num_observed", C.c_int64),
        ("depth_count", C.c_int64),
        ("color_count", C.c_int64),
        ("depth_abs", C.c_double),
        ("depth_sq", C.c_double),
        ("color_abs", C.c_int64 * 3),
        ("color_sq", C.c_int64 * 3),
    ]


class I3DRasterInfo(C.Structure, _Dictable):
    _fields_ = [
        ("num_views", C.c_int64),
        ("num_faces", C.c_int64),
        ("num_pairs", C.c_int64),
        ("num_straddling", C.c_int64),
        ("num_behind", C.c_int64),
        ("num_tests", C.c_int64),
        ("num_covered", C.c_int64),
        ("ms_rays", C.c_double),
        ("ms_faces", C.c_double),
        ("ms_shade", C.c_double),
    ]


TRACK_LEVELS = 4          # entries of I3DTrackParams::iterations
TRACK_STATUS = {0: "tracked", 1: "too few correspondences", 2: "not positive definite", 3: "non-finite", 4: "anchored"}


class I3DTrackParams(C.Structure, _Dictable):
    _fields_ = [
        ("sdf_source", C.c_int32),
        ("num_levels", C.c_int32),
        ("iterations", C.c_int32 * TRACK_LEVELS),
        ("max_distance", C.c_float),
        ("min_normal_cos", C.c_float),
        ("min_correspondences", C.c_int32),
        ("reserved", C.c_int32),
    ]


class I3DTrackInfo(C.Structure, _Dictable):
    _fields_ = [
        ("status", C.c_int32),
        ("iterations", C.c_int32),
        ("correspondences", C.c_int64),
        ("residual_sq", C.c_double),
        ("update_norm", C.c_double),
        ("initial", I3DRenderStats),
    ]

    def as_dict(self):
        out = _Dictable.as_dict(self)
        out["initial"] = self.initial.as_dict()
        return out


class I3DTrackColorParams(C.Structure, _Dictable):
    _fields_ = [
        ("weight", C.c_float * TRACK_LEVELS),
        ("max_color_diff", C.c_float),
        ("min_color_gradient", C.c_float),
        ("norm_radius", C.c_int32),
        ("norm_eps", C.c_float),
    ]


class I3DTrackColorInfo(C.Structure, _Dictable):
    _fields_ = [
        ("first_rows", C.c_int64),
        ("first_residual_sq", C.c_double),
        ("last_rows", C.c_int64),
        ("last_residual_sq", C.c_double),
    ]
