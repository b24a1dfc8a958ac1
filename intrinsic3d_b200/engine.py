"""Python host-side binding of the C-ABI in include/i3d_c_api.h (libi3d_b200.so).

This is plumbing for tests and bench.py: it passes HOST numpy buffers through the same
extern "C" entry points a C++ caller (include/nv/refinement/ shims) uses.  There is no CPU
fallback: if the CUDA library is missing or no sm_90 (H100) device is present, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .ctypes_defs import (DISTANCE_MAX_THRESHOLDS, GRID_FROM_MESH_SOURCES, RASTER_COLORS, RASTER_PLANES, REGISTER_MAX_STAGES, RENDER_PLANES, SH_SOURCES,
                          I3DDistanceInfo, I3DRegisterInfo, I3DRegisterParams,
                          I3DDistanceParams, I3DGridFromMeshInfo, I3DGridFromMeshParams, I3DFusionCamera, I3DFusionParams, I3DIntrinsicTextureInfo,
                          I3DIntrinsicTextureParams, I3DIterInfo, I3DShLighting,
                          I3DLightingInfo, I3DLightingParams, I3DMeshInfo, I3DMeshParams, I3DParams, I3DRasterCamera, I3DRasterInfo,
                          I3DRasterParams, I3DRasterStats, I3DRenderParams, I3DRenderStats, I3DSimplifyInfo, I3DSimplifyParams, I3DTextureInfo,
                          I3DTextureParams, I3DTrackColorInfo, I3DTrackColorParams, I3DTrackInfo, I3DTrackParams, TRACK_LEVELS)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("I3D_LIB", os.path.join(_HERE, "libi3d_b200.so"))   # I3D_LIB: A/B builds of the same library
_LIB = None

EXPORTED_SYMBOLS = [
    "i3d_abi_version", "i3d_sizeof_params", "i3d_sizeof_iter_info", "i3d_default_params",
    "i3d_engine_create", "i3d_engine_destroy", "i3d_last_error",
    "i3d_upload_grid", "i3d_upload_voxel_params", "i3d_upload_frames", "i3d_set_camera", "i3d_set_sh",
    "i3d_gn_iteration", "i3d_download_state",
    "i3d_sizeof_lighting_params", "i3d_sizeof_lighting_info", "i3d_default_lighting_params", "i3d_estimate_lighting",
    "i3d_lighting_num_subvolumes", "i3d_download_lighting", "i3d_download_voxel_sh",
    "i3d_upload_color_frames", "i3d_recompute_colors", "i3d_download_colors",
    "i3d_num_voxels", "i3d_clear_voxels_outside_thin_shell", "i3d_upsample_grid", "i3d_download_grid",
    "i3d_sizeof_fusion_params", "i3d_default_fusion_params", "i3d_fusion_begin", "i3d_fusion_integrate", "i3d_fusion_finish",
    "i3d_keyframe_scores", "i3d_upload_rgbd_frames", "i3d_use_rgbd_level",
    "i3d_sensor_frames_begin", "i3d_sensor_frames_add", "i3d_sensor_num_frames", "i3d_sensor_keyframe_scores", "i3d_fusion_integrate_sensor",
    "i3d_select_rgbd_frames",
    "i3d_sizeof_mesh_info", "i3d_extract_mesh", "i3d_download_mesh", "i3d_extract_mesh_colored", "i3d_mode_colors",
    "i3d_sizeof_simplify_params", "i3d_sizeof_simplify_info", "i3d_simplify_mesh",
    "i3d_sizeof_texture_params", "i3d_sizeof_texture_info", "i3d_default_texture_params", "i3d_bake_texture", "i3d_download_texture",
    "i3d_sizeof_sh_lighting", "i3d_sizeof_intrinsic_texture_params", "i3d_sizeof_intrinsic_texture_info", "i3d_default_sh_lighting",
    "i3d_default_intrinsic_texture_params", "i3d_decompose_texture", "i3d_download_intrinsic_texture", "i3d_set_relight",
    "i3d_sizeof_distance_params", "i3d_sizeof_distance_info", "i3d_default_distance_params", "i3d_upload_reference_mesh",
    "i3d_surface_distance", "i3d_download_surface_distance", "i3d_debug_set_keep_distance_samples", "i3d_debug_get_distance_samples",
    "i3d_sizeof_register_params", "i3d_sizeof_register_info", "i3d_default_register_params", "i3d_register_reference_mesh",
    "i3d_transform_reference_mesh", "i3d_debug_get_register_systems",
    "i3d_sizeof_grid_from_mesh_params", "i3d_sizeof_grid_from_mesh_info", "i3d_default_grid_from_mesh_params", "i3d_grid_from_mesh",
    "i3d_debug_get_grid_from_mesh_voxels",
    "i3d_sizeof_render_params", "i3d_sizeof_render_stats", "i3d_default_render_params", "i3d_render_keyframes", "i3d_download_render",
    "i3d_debug_set_render_skip",
    "i3d_sizeof_raster_params", "i3d_sizeof_raster_camera", "i3d_sizeof_raster_stats", "i3d_sizeof_raster_info", "i3d_default_raster_params",
    "i3d_rasterize_keyframes", "i3d_rasterize_views", "i3d_download_raster", "i3d_debug_set_raster_binning",
    "i3d_debug_set_raster_batch",
    "i3d_sizeof_track_params", "i3d_sizeof_track_info", "i3d_default_track_params", "i3d_track_sensor_frames", "i3d_debug_get_track_system",
    "i3d_debug_get_track_planes", "i3d_fusion_track_sensor_frames", "i3d_fusion_track_and_integrate_sensor",
    "i3d_sizeof_track_color_params", "i3d_sizeof_track_color_info", "i3d_default_track_color_params", "i3d_track_sensor_frames_rgbd",
    "i3d_fusion_track_sensor_frames_rgbd", "i3d_fusion_track_and_integrate_sensor_rgbd", "i3d_debug_get_track_color_planes",
    "i3d_debug_get_track_color_system", "i3d_track_sensor_frames_rgbd_ref", "i3d_fusion_track_sensor_frames_rgbd_ref",
    "i3d_fusion_track_and_integrate_sensor_rgbd_ref", "i3d_debug_get_track_reference_planes", "i3d_default_track_color_ref_params",
    "i3d_default_track_color_lni_params",
    "i3d_comm_unique_id", "i3d_comm_init", "i3d_comm_p2p_export", "i3d_comm_p2p_connect", "i3d_set_shard",
    "i3d_phase_ms", "i3d_phase_count", "i3d_debug_set_kernel_timers", "i3d_debug_num_slots", "i3d_debug_set_keep_raw_jacobian",
    "i3d_debug_get_rows", "i3d_debug_get_observations", "i3d_debug_get_step", "i3d_debug_get_pcg_vectors", "i3d_debug_get_normal_equations",
    "i3d_debug_apply_operator", "i3d_debug_fusion_num_voxels", "i3d_debug_get_fusion_volume", "i3d_debug_get_frames",
]
KEYFRAME_CHUNK = 32       # I3D_KEYFRAME_CHUNK of include/i3d_c_api.h: frames scored per device pass
# SDFVisualization's colour mode strings -> I3D_MESH_COLOR_* of include/i3d_types.h
COLOR_MODES = {"": 0, "normals": 1, "lap": 2, "lum": 3, "lum_grad": 4, "albedo": 5, "shading_sv": 6, "shading_sv_const": 7, "chroma": 8}


def load_library():
    """Loads libi3d_b200.so.  Raises (never falls back) when the CUDA extension is missing."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: build it with intrinsic3d_b200/csrc/build.sh "
                           "(__graft_entry__.build()); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    L.i3d_abi_version.restype = C.c_int
    L.i3d_sizeof_params.restype = C.c_uint64
    L.i3d_sizeof_iter_info.restype = C.c_uint64
    L.i3d_last_error.restype = C.c_char_p
    L.i3d_last_error.argtypes = [C.c_void_p]
    L.i3d_phase_ms.restype = C.c_double
    L.i3d_phase_ms.argtypes = [C.c_void_p, C.c_char_p]
    L.i3d_phase_count.restype = C.c_int64
    L.i3d_phase_count.argtypes = [C.c_void_p, C.c_char_p]
    L.i3d_debug_num_slots.restype = C.c_int64
    L.i3d_debug_num_slots.argtypes = [C.c_void_p]
    L.i3d_sizeof_lighting_params.restype = C.c_uint64
    L.i3d_sizeof_lighting_info.restype = C.c_uint64
    L.i3d_lighting_num_subvolumes.restype = C.c_int64
    L.i3d_lighting_num_subvolumes.argtypes = [C.c_void_p]
    L.i3d_num_voxels.restype = C.c_int64
    L.i3d_num_voxels.argtypes = [C.c_void_p]
    L.i3d_sizeof_fusion_params.restype = C.c_uint64
    L.i3d_debug_fusion_num_voxels.restype = C.c_int64
    L.i3d_debug_fusion_num_voxels.argtypes = [C.c_void_p]
    if L.i3d_sizeof_params() != C.sizeof(I3DParams) or L.i3d_sizeof_iter_info() != C.sizeof(I3DIterInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so")
    if L.i3d_sizeof_lighting_params() != C.sizeof(I3DLightingParams) or L.i3d_sizeof_lighting_info() != C.sizeof(I3DLightingInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (lighting structs)")
    if L.i3d_sizeof_fusion_params() != C.sizeof(I3DFusionParams):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (fusion params)")
    L.i3d_sizeof_mesh_info.restype = C.c_uint64
    if L.i3d_sizeof_mesh_info() != C.sizeof(I3DMeshInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (mesh info)")
    L.i3d_extract_mesh_colored.restype = C.c_int
    L.i3d_extract_mesh_colored.argtypes = [C.c_void_p, C.POINTER(I3DMeshParams), C.c_int32, C.POINTER(I3DMeshInfo)]
    L.i3d_sizeof_simplify_params.restype = C.c_uint64
    L.i3d_sizeof_simplify_info.restype = C.c_uint64
    if L.i3d_sizeof_simplify_params() != C.sizeof(I3DSimplifyParams) or L.i3d_sizeof_simplify_info() != C.sizeof(I3DSimplifyInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (simplify structs)")
    L.i3d_simplify_mesh.restype = C.c_int
    L.i3d_simplify_mesh.argtypes = [C.c_void_p, C.POINTER(I3DSimplifyParams), C.POINTER(I3DSimplifyInfo)]
    L.i3d_sizeof_texture_params.restype = C.c_uint64
    L.i3d_sizeof_texture_info.restype = C.c_uint64
    if L.i3d_sizeof_texture_params() != C.sizeof(I3DTextureParams) or L.i3d_sizeof_texture_info() != C.sizeof(I3DTextureInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (texture structs)")
    L.i3d_default_texture_params.restype = None
    L.i3d_default_texture_params.argtypes = [C.POINTER(I3DTextureParams)]
    L.i3d_bake_texture.restype = C.c_int
    L.i3d_bake_texture.argtypes = [C.c_void_p, C.POINTER(I3DTextureParams), C.POINTER(C.c_float), C.POINTER(I3DTextureInfo)]
    L.i3d_download_texture.restype = C.c_int
    L.i3d_download_texture.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_float)]
    for fn in (L.i3d_sizeof_sh_lighting, L.i3d_sizeof_intrinsic_texture_params, L.i3d_sizeof_intrinsic_texture_info):
        fn.restype = C.c_uint64
    if (L.i3d_sizeof_sh_lighting() != C.sizeof(I3DShLighting) or L.i3d_sizeof_intrinsic_texture_params() != C.sizeof(I3DIntrinsicTextureParams)
            or L.i3d_sizeof_intrinsic_texture_info() != C.sizeof(I3DIntrinsicTextureInfo)):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (intrinsic texture structs)")
    L.i3d_default_sh_lighting.restype = None
    L.i3d_default_sh_lighting.argtypes = [C.POINTER(I3DShLighting)]
    L.i3d_default_intrinsic_texture_params.restype = None
    L.i3d_default_intrinsic_texture_params.argtypes = [C.POINTER(I3DIntrinsicTextureParams)]
    L.i3d_decompose_texture.restype = C.c_int
    L.i3d_decompose_texture.argtypes = [C.c_void_p, C.POINTER(I3DIntrinsicTextureParams), C.POINTER(I3DIntrinsicTextureInfo)]
    L.i3d_download_intrinsic_texture.restype = C.c_int
    L.i3d_download_intrinsic_texture.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.i3d_set_relight.restype = C.c_int
    L.i3d_set_relight.argtypes = [C.c_void_p, C.POINTER(I3DShLighting)]
    L.i3d_sizeof_distance_params.restype = C.c_uint64
    L.i3d_sizeof_distance_info.restype = C.c_uint64
    if L.i3d_sizeof_distance_params() != C.sizeof(I3DDistanceParams) or L.i3d_sizeof_distance_info() != C.sizeof(I3DDistanceInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (distance structs)")
    L.i3d_default_distance_params.restype = None
    L.i3d_default_distance_params.argtypes = [C.POINTER(I3DDistanceParams)]
    L.i3d_upload_reference_mesh.restype = C.c_int
    L.i3d_upload_reference_mesh.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_float), C.c_int64, C.POINTER(C.c_int32)]
    L.i3d_surface_distance.restype = C.c_int
    L.i3d_surface_distance.argtypes = [C.c_void_p, C.POINTER(I3DDistanceParams), C.POINTER(I3DDistanceInfo)]
    L.i3d_download_surface_distance.restype = C.c_int
    L.i3d_download_surface_distance.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int32)]
    L.i3d_debug_set_keep_distance_samples.restype = C.c_int
    L.i3d_debug_set_keep_distance_samples.argtypes = [C.c_void_p, C.c_int]
    L.i3d_debug_get_distance_samples.restype = C.c_int
    L.i3d_debug_get_distance_samples.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int32)]
    L.i3d_sizeof_register_params.restype = C.c_uint64
    L.i3d_sizeof_register_info.restype = C.c_uint64
    if L.i3d_sizeof_register_params() != C.sizeof(I3DRegisterParams) or L.i3d_sizeof_register_info() != C.sizeof(I3DRegisterInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (register structs)")
    L.i3d_default_register_params.restype = None
    L.i3d_default_register_params.argtypes = [C.POINTER(I3DRegisterParams)]
    L.i3d_register_reference_mesh.restype = C.c_int
    L.i3d_register_reference_mesh.argtypes = [C.c_void_p, C.POINTER(I3DRegisterParams), C.POINTER(C.c_double), C.POINTER(C.c_double),
                                              C.POINTER(I3DRegisterInfo)]
    L.i3d_transform_reference_mesh.restype = C.c_int
    L.i3d_transform_reference_mesh.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    L.i3d_debug_get_register_systems.restype = C.c_int
    L.i3d_debug_get_register_systems.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_double),
                                                 C.POINTER(C.c_int32)]
    L.i3d_sizeof_grid_from_mesh_params.restype = C.c_uint64
    L.i3d_sizeof_grid_from_mesh_info.restype = C.c_uint64
    if L.i3d_sizeof_grid_from_mesh_params() != C.sizeof(I3DGridFromMeshParams) or L.i3d_sizeof_grid_from_mesh_info() != C.sizeof(I3DGridFromMeshInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (grid-from-mesh structs)")
    L.i3d_default_grid_from_mesh_params.restype = None
    L.i3d_default_grid_from_mesh_params.argtypes = [C.POINTER(I3DGridFromMeshParams)]
    L.i3d_grid_from_mesh.restype = C.c_int
    L.i3d_grid_from_mesh.argtypes = [C.c_void_p, C.POINTER(I3DGridFromMeshParams), C.POINTER(I3DGridFromMeshInfo)]
    L.i3d_debug_get_grid_from_mesh_voxels.restype = C.c_int
    L.i3d_debug_get_grid_from_mesh_voxels.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int8)]
    L.i3d_mode_colors.restype = C.c_int
    L.i3d_mode_colors.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_uint8)]
    L.i3d_sensor_num_frames.restype = C.c_int32
    L.i3d_sensor_num_frames.argtypes = [C.c_void_p]
    L.i3d_sizeof_render_params.restype = C.c_uint64
    L.i3d_sizeof_render_stats.restype = C.c_uint64
    if L.i3d_sizeof_render_params() != C.sizeof(I3DRenderParams) or L.i3d_sizeof_render_stats() != C.sizeof(I3DRenderStats):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (render structs)")
    L.i3d_render_keyframes.restype = C.c_int
    L.i3d_render_keyframes.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(I3DRenderParams), C.POINTER(I3DRenderStats)]
    L.i3d_download_render.restype = C.c_int
    L.i3d_download_render.argtypes = [C.c_void_p] + [C.POINTER(C.c_float)] * 5
    for fn in (L.i3d_sizeof_raster_params, L.i3d_sizeof_raster_camera, L.i3d_sizeof_raster_stats, L.i3d_sizeof_raster_info):
        fn.restype = C.c_uint64
    if (L.i3d_sizeof_raster_params() != C.sizeof(I3DRasterParams) or L.i3d_sizeof_raster_camera() != C.sizeof(I3DRasterCamera)
            or L.i3d_sizeof_raster_stats() != C.sizeof(I3DRasterStats) or L.i3d_sizeof_raster_info() != C.sizeof(I3DRasterInfo)):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (raster structs)")
    L.i3d_default_raster_params.restype = None
    L.i3d_default_raster_params.argtypes = [C.POINTER(I3DRasterParams)]
    L.i3d_rasterize_keyframes.restype = C.c_int
    L.i3d_rasterize_keyframes.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(I3DRasterParams), C.POINTER(I3DRasterStats),
                                          C.POINTER(I3DRasterInfo)]
    L.i3d_rasterize_views.restype = C.c_int
    L.i3d_rasterize_views.argtypes = [C.c_void_p, C.c_int32, C.POINTER(I3DRasterCamera), C.POINTER(C.c_float), C.POINTER(I3DRasterParams),
                                      C.POINTER(I3DRasterInfo)]
    L.i3d_download_raster.restype = C.c_int
    L.i3d_download_raster.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                      C.POINTER(C.c_uint8)]
    L.i3d_debug_set_raster_binning.restype = C.c_int
    L.i3d_debug_set_raster_binning.argtypes = [C.c_void_p, C.c_int]
    L.i3d_debug_set_raster_batch.restype = C.c_int
    L.i3d_debug_set_raster_batch.argtypes = [C.c_void_p, C.c_int]
    L.i3d_sizeof_track_params.restype = C.c_uint64
    L.i3d_sizeof_track_info.restype = C.c_uint64
    if L.i3d_sizeof_track_params() != C.sizeof(I3DTrackParams) or L.i3d_sizeof_track_info() != C.sizeof(I3DTrackInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (track structs)")
    L.i3d_track_sensor_frames.restype = C.c_int
    L.i3d_track_sensor_frames.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(I3DTrackParams),
                                          C.POINTER(C.c_double), C.POINTER(I3DTrackInfo)]
    for fn in (L.i3d_fusion_track_sensor_frames, L.i3d_fusion_track_and_integrate_sensor):
        fn.restype = C.c_int
        fn.argtypes = L.i3d_track_sensor_frames.argtypes
    L.i3d_debug_get_track_system.restype = C.c_int
    L.i3d_debug_get_track_system.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    L.i3d_debug_get_track_planes.restype = C.c_int
    L.i3d_debug_get_track_planes.argtypes = [C.c_void_p, C.c_int32] + [C.POINTER(C.c_float)] * 4 + [C.POINTER(C.c_uint8), C.POINTER(C.c_int32)]
    L.i3d_sizeof_track_color_params.restype = C.c_uint64
    L.i3d_sizeof_track_color_info.restype = C.c_uint64
    if L.i3d_sizeof_track_color_params() != C.sizeof(I3DTrackColorParams) or L.i3d_sizeof_track_color_info() != C.sizeof(I3DTrackColorInfo):
        raise RuntimeError("ABI mismatch between ctypes_defs.py and libi3d_b200.so (track colour structs)")
    for fn in (L.i3d_track_sensor_frames_rgbd, L.i3d_fusion_track_sensor_frames_rgbd, L.i3d_fusion_track_and_integrate_sensor_rgbd):
        fn.restype = C.c_int
        fn.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(I3DTrackParams),
                       C.POINTER(I3DTrackColorParams), C.POINTER(C.c_double), C.POINTER(I3DTrackInfo), C.POINTER(I3DTrackColorInfo)]
    L.i3d_debug_get_track_color_planes.restype = C.c_int
    L.i3d_debug_get_track_color_planes.argtypes = [C.c_void_p, C.c_int32] + [C.POINTER(C.c_float)] * 4 + [C.POINTER(C.c_int32)]
    L.i3d_debug_get_track_color_system.restype = C.c_int
    L.i3d_debug_get_track_color_system.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    for fn in (L.i3d_track_sensor_frames_rgbd_ref, L.i3d_fusion_track_sensor_frames_rgbd_ref):
        fn.restype = C.c_int
        fn.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_double),
                       C.POINTER(I3DTrackParams), C.POINTER(I3DTrackColorParams), C.POINTER(C.c_double), C.POINTER(I3DTrackInfo),
                       C.POINTER(I3DTrackColorInfo)]
    L.i3d_fusion_track_and_integrate_sensor_rgbd_ref.restype = C.c_int
    L.i3d_fusion_track_and_integrate_sensor_rgbd_ref.argtypes = L.i3d_fusion_track_and_integrate_sensor_rgbd.argtypes
    L.i3d_debug_get_track_reference_planes.restype = C.c_int
    L.i3d_debug_get_track_reference_planes.argtypes = [C.c_void_p, C.c_int32] + [C.POINTER(C.c_float)] * 3 + [C.POINTER(C.c_int32)]
    _LIB = L
    return L


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def default_params() -> I3DParams:
    p = I3DParams()
    load_library().i3d_default_params(C.byref(p))
    return p


def default_lighting_params() -> I3DLightingParams:
    p = I3DLightingParams()
    load_library().i3d_default_lighting_params(C.byref(p))
    return p


def default_fusion_params() -> I3DFusionParams:
    p = I3DFusionParams()
    load_library().i3d_default_fusion_params(C.byref(p))
    return p


def default_track_params() -> I3DTrackParams:
    p = I3DTrackParams()
    load_library().i3d_default_track_params(C.byref(p))
    return p


def default_track_color_params() -> I3DTrackColorParams:
    p = I3DTrackColorParams()
    load_library().i3d_default_track_color_params(C.byref(p))
    return p


def default_track_color_ref_params() -> I3DTrackColorParams:
    p = I3DTrackColorParams()
    load_library().i3d_default_track_color_ref_params(C.byref(p))
    return p


def default_track_color_lni_params() -> I3DTrackColorParams:
    """the _ref calls' parameters with locally normalised intensity (norm_radius > 0, DESIGN.md §6r)"""
    p = I3DTrackColorParams()
    load_library().i3d_default_track_color_lni_params(C.byref(p))
    return p


def sh_lighting(sh=None) -> I3DShLighting:
    """The I3DShLighting of sh: None for the subvolume SH of the last lighting estimate, else nine coefficients (the order of the lighting
    estimate) used everywhere."""
    if sh is None:
        return I3DShLighting(SH_SOURCES["estimate"], 0, (C.c_float * 9)())
    v = np.asarray(sh, np.float32).reshape(-1)
    if v.shape != (9,):
        raise ValueError(f"sh must hold 9 coefficients, got {v.size}")
    return I3DShLighting(SH_SOURCES["global"], 0, (C.c_float * 9)(*[float(x) for x in v]))


def default_texture_params() -> I3DTextureParams:
    p = I3DTextureParams()
    load_library().i3d_default_texture_params(C.byref(p))
    return p


def default_distance_params() -> I3DDistanceParams:
    p = I3DDistanceParams()
    load_library().i3d_default_distance_params(C.byref(p))
    return p


def default_register_params() -> I3DRegisterParams:
    p = I3DRegisterParams()
    load_library().i3d_default_register_params(C.byref(p))
    return p


def fusion_camera(cam) -> I3DFusionCamera:
    """(W, H, fx, fy, cx, cy) -> I3DFusionCamera."""
    W, H, fx, fy, cx, cy = cam
    return I3DFusionCamera(int(W), int(H), float(fx), float(fy), float(cx), float(cy))


class Engine:
    """One GPU-resident problem: grid + frames + camera + SH; gn_iteration() = one outer GN iteration."""

    def __init__(self, device: int = 0):
        self.L = load_library()
        h = C.c_void_p()
        rc = self.L.i3d_engine_create(C.c_int(device), C.byref(h))
        if rc != 0:
            raise RuntimeError("i3d_engine_create failed: " + self.L.i3d_last_error(None).decode())
        self.h = h
        self.n = 0
        self.F = 0

    def close(self):
        if getattr(self, "h", None):
            self.L.i3d_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.i3d_last_error(self.h).decode())

    # ---- uploads (host buffers; copied during the call) -------------------------------------
    def upload_grid(self, xyz, sdf0, sdf_refined, albedo, weight, rgb, voxel_size):
        xyz = np.ascontiguousarray(xyz, np.int32)
        n = int(xyz.shape[0])
        a = [np.ascontiguousarray(sdf0, np.float64), np.ascontiguousarray(sdf_refined, np.float64),
             np.ascontiguousarray(albedo, np.float64), np.ascontiguousarray(weight, np.float32),
             np.ascontiguousarray(rgb, np.uint8)]
        self._check(self.L.i3d_upload_grid(self.h, C.c_int64(n), _p(xyz, C.c_int32), _p(a[0], C.c_double), _p(a[1], C.c_double),
                                           _p(a[2], C.c_double), _p(a[3], C.c_float), _p(a[4], C.c_uint8), C.c_float(float(voxel_size))))
        self.n = n

    def upload_voxel_params(self, sdf_refined, albedo):
        s = np.ascontiguousarray(sdf_refined, np.float64)
        a = np.ascontiguousarray(albedo, np.float64)
        self._check(self.L.i3d_upload_voxel_params(self.h, _p(s, C.c_double), _p(a, C.c_double)))

    def upload_frames(self, lum, depth, pyr_scale=1.0):
        lum = np.ascontiguousarray(lum, np.float32)
        depth = np.ascontiguousarray(depth, np.float32)
        F, H, W = lum.shape
        self._check(self.L.i3d_upload_frames(self.h, C.c_int32(F), C.c_int32(W), C.c_int32(H), _p(lum, C.c_float), _p(depth, C.c_float),
                                             C.c_double(float(pyr_scale))))
        self.F = F
        self.frame_size = (W, H)

    def set_camera(self, poses, intr, dist):
        poses = np.ascontiguousarray(poses, np.float64)
        intr = np.ascontiguousarray(intr, np.float64)
        dist = np.ascontiguousarray(dist, np.float64)
        self._check(self.L.i3d_set_camera(self.h, _p(poses, C.c_double), _p(intr, C.c_double), _p(dist, C.c_double)))

    def set_sh(self, sh):
        sh = np.ascontiguousarray(sh, np.float64)
        assert sh.shape == (self.n, 9)
        self._check(self.L.i3d_set_sh(self.h, _p(sh, C.c_double)))

    def load_scene(self, s):
        self.upload_grid(s["xyz"], s["sdf0"], s["sdf_refined"], s["albedo"], s["weight"], s["rgb"], s["voxel_size"])
        self.upload_frames(s["lum"], s["depth"], s.get("pyr_scale", 1.0))
        self.set_camera(s["poses"], s["intr"], s["dist"])
        self.set_sh(s["sh"])

    # ---- compute ----------------------------------------------------------------------------
    def gn_iteration(self, params: I3DParams) -> I3DIterInfo:
        info = I3DIterInfo()
        self._check(self.L.i3d_gn_iteration(self.h, C.byref(params), C.byref(info)))
        return info

    # ---- SVSH lighting (LightingSVSH::estimate + computeVoxelShCoeffs) -----------------------
    def estimate_lighting(self, params: I3DLightingParams) -> I3DLightingInfo:
        """Estimates the subvolume SH on the uploaded grid and leaves the per-voxel blend as the engine's `sh` input."""
        info = I3DLightingInfo()
        self._check(self.L.i3d_estimate_lighting(self.h, C.byref(params), C.byref(info)))
        return info

    def download_lighting(self):
        S = int(self.L.i3d_lighting_num_subvolumes(self.h))
        idx = np.empty((S, 3), np.int32)
        sh = np.empty((S, 9), np.float64)
        self._check(self.L.i3d_download_lighting(self.h, _p(idx, C.c_int32), _p(sh, C.c_double)))
        return idx, sh

    def download_voxel_sh(self):
        sh = np.empty((self.n, 9), np.float64)
        has = np.empty(self.n, np.uint8)
        self._check(self.L.i3d_download_voxel_sh(self.h, _p(sh, C.c_double), _p(has, C.c_uint8)))
        return sh, has

    # ---- voxel recolouring (Intrinsic3D::recomputeColors) ------------------------------------
    def upload_color_frames(self, bgr):
        bgr = np.ascontiguousarray(bgr, np.uint8)
        assert bgr.ndim == 4 and bgr.shape[0] == self.F and bgr.shape[3] == 3
        self._check(self.L.i3d_upload_color_frames(self.h, _p(bgr, C.c_uint8)))

    def recompute_colors(self, max_occlusion_distance: float = 0.02, max_num_observations: int = 5, pose_rt=None):
        """Returns (voxels recoloured, observations with weight > 0).  pose_rt: optional float32 [F, 12] (R row-major | t)."""
        a, b = C.c_int64(0), C.c_int64(0)
        if pose_rt is not None:
            pose_rt = np.ascontiguousarray(pose_rt, np.float32)
            assert pose_rt.shape == (self.F, 12)
        self._check(self.L.i3d_recompute_colors(self.h, _p(pose_rt, C.c_float), C.c_float(max_occlusion_distance), C.c_int32(max_num_observations),
                                                C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def download_colors(self):
        rgb = np.empty((self.n, 3), np.uint8)
        self._check(self.L.i3d_download_colors(self.h, _p(rgb, C.c_uint8)))
        return rgb

    # ---- grid-level transitions (SDFAlgorithms::clearVoxelsOutsideThinShell / upsample) -------
    def clear_voxels_outside_thin_shell(self, thres_shell: float) -> int:
        m = C.c_int64(0)
        self._check(self.L.i3d_clear_voxels_outside_thin_shell(self.h, C.c_double(thres_shell), C.byref(m)))
        self.n = int(m.value)
        return self.n

    def upsample_grid(self) -> int:
        m = C.c_int64(0)
        self._check(self.L.i3d_upsample_grid(self.h, C.byref(m)))
        self.n = int(m.value)
        return self.n

    def download_grid(self):
        n = int(self.L.i3d_num_voxels(self.h))
        out = dict(xyz=np.empty((n, 3), np.int32), sdf0=np.empty(n, np.float64), sdf_refined=np.empty(n, np.float64), albedo=np.empty(n, np.float64),
                   weight=np.empty(n, np.float32), rgb=np.empty((n, 3), np.uint8))
        vs = C.c_float(0)
        self._check(self.L.i3d_download_grid(self.h, _p(out["xyz"], C.c_int32), _p(out["sdf0"], C.c_double), _p(out["sdf_refined"], C.c_double),
                                             _p(out["albedo"], C.c_double), _p(out["weight"], C.c_float), _p(out["rgb"], C.c_uint8), C.byref(vs)))
        out["voxel_size"] = np.float32(vs.value)
        return out

    # ---- RGB-D fusion (AppFusion::fuseSDF) -------------------------------------------------------
    def fusion_begin(self, params: I3DFusionParams):
        self._check(self.L.i3d_fusion_begin(self.h, C.byref(params)))

    def fusion_integrate(self, depth_cam, depth, color_cam, bgr, pose_cam_to_world, pose_world_to_cam):
        """depth float32 [F, Hd, Wd] metres; bgr uint8 [F, Hc, Wc, 3]; cameras (W, H, fx, fy, cx, cy); poses float32 [F, 12] (R row-major | t)."""
        depth = np.ascontiguousarray(depth, np.float32)
        bgr = np.ascontiguousarray(bgr, np.uint8)
        c2w = np.ascontiguousarray(pose_cam_to_world, np.float32)
        w2c = np.ascontiguousarray(pose_world_to_cam, np.float32)
        F = int(depth.shape[0])
        dc, cc = fusion_camera(depth_cam), fusion_camera(color_cam)
        assert depth.shape == (F, dc.height, dc.width) and bgr.shape == (F, cc.height, cc.width, 3)
        assert c2w.shape == (F, 12) and w2c.shape == (F, 12)
        self._check(self.L.i3d_fusion_integrate(self.h, C.c_int32(F), C.byref(dc), _p(depth, C.c_float), C.byref(cc), _p(bgr, C.c_uint8),
                                                _p(c2w, C.c_float), _p(w2c, C.c_float)))

    def fusion_finish(self) -> int:
        """correctSDF, clearInvalidVoxels, convert; the result becomes the engine's grid.  Returns its voxel count."""
        m = C.c_int64(0)
        self._check(self.L.i3d_fusion_finish(self.h, C.byref(m)))
        self.n = int(m.value)
        return self.n

    def fusion_volume(self):
        """The fusion volume in progress in canonical order: xyz, sdf (float32), weight, rgb."""
        n = int(self.L.i3d_debug_fusion_num_voxels(self.h))
        out = dict(xyz=np.empty((n, 3), np.int32), sdf=np.empty(n, np.float32), weight=np.empty(n, np.float32), rgb=np.empty((n, 3), np.uint8))
        self._check(self.L.i3d_debug_get_fusion_volume(self.h, _p(out["xyz"], C.c_int32), _p(out["sdf"], C.c_float), _p(out["weight"], C.c_float),
                                                       _p(out["rgb"], C.c_uint8)))
        return out

    # ---- surface extraction (MarchingCubes::extractSurface + MeshUtil) ------------------------------------------------------
    MESH_SOURCES = {"fused": 0, "refined": 1}

    def _mesh_source(self, source):
        if source not in self.MESH_SOURCES:
            raise ValueError(f"source must be one of {sorted(self.MESH_SOURCES)}, got {source!r}")
        return self.MESH_SOURCES[source]

    @staticmethod
    def _color_mode(mode):
        if mode not in COLOR_MODES:
            raise ValueError(f"colour mode must be one of {sorted(COLOR_MODES)} (the subvolume modes are not supported), got {mode!r}")
        return COLOR_MODES[mode]

    def extract_mesh(self, source: str = "refined", largest_component_only: bool = False, color_mode: str = ""):
        """The grid's zero level set as a coloured triangle mesh, extracted on the device: source "fused" meshes sdf0 (as AppFusion does),
        "refined" the refined sdf (as AppIntrinsic3D::onSDFRefined does).  color_mode is a mode string of SDFVisualization::colorize:
        "" (the voxel colours), "normals", "lap", "lum", "lum_grad", "albedo", "shading_sv", "shading_sv_const" or "chroma"; the shading
        modes need a lighting estimate of the current grid (estimate_lighting).  largest_component_only keeps the face-connected
        component with the most faces (output_mesh_largest_comp_only).  Returns a dict with vertices float32 [V, 3] (metres), colors
        uint8 [V, 3], faces int32 [F, 3] and info (I3DMeshInfo: counts per stage, device ms per stage; the colour pass is
        phase_ms("mesh_colorize")).  Write it with mesh.save_ply."""
        src = self._mesh_source(source)
        mode = self._color_mode(color_mode)
        prm = I3DMeshParams(src, 1 if largest_component_only else 0)
        info = I3DMeshInfo()
        if mode == 0:
            self._check(self.L.i3d_extract_mesh(self.h, C.byref(prm), C.byref(info)))
        else:
            self._check(self.L.i3d_extract_mesh_colored(self.h, C.byref(prm), mode, C.byref(info)))
        return self._download_mesh(info)

    def _download_mesh(self, info):
        V, F = int(info.num_vertices), int(info.num_faces)
        out = dict(vertices=np.empty((V, 3), np.float32), colors=np.empty((V, 3), np.uint8), faces=np.empty((F, 3), np.int32), info=info)
        self._check(self.L.i3d_download_mesh(self.h, _p(out["vertices"], C.c_float), _p(out["colors"], C.c_uint8), _p(out["faces"], C.c_int32)))
        return out

    def simplify_mesh(self, cell_size: float):
        """Simplifies the resident mesh (the last extract_mesh or simplify_mesh of the current grid) on the device by quadric-error vertex
        clustering (DESIGN.md §6s): the vertices in each world-aligned cube of edge cell_size (metres) become one vertex placed by the
        summed face-plane quadrics, and the faces that collapse, repeat or degenerate go.  The result replaces the resident mesh, so a
        second call gives a coarser mesh.  Returns the dict extract_mesh returns, with info an I3DSimplifyInfo (clusters, dropped faces
        by reason, counts of the result, device ms per stage)."""
        info = I3DSimplifyInfo()
        self._check(self.L.i3d_simplify_mesh(self.h, C.byref(I3DSimplifyParams(float(cell_size), 0)), C.byref(info)))
        return self._download_mesh(info)

    def bake_texture(self, texels_per_face: int = 12, max_occlusion_distance: float = 0.02, max_num_observations: int = 5, pose_rt=None):
        """Bakes the keyframes' colour into a texture atlas of the resident mesh (the last extract_mesh or simplify_mesh) on the device
        (DESIGN.md §6t): faces 2c and 2c+1 share a cell of texels_per_face x texels_per_face texels, and every texel a face owns gets
        recompute_colors' colour at its 3-D point, or the barycentric blend of the vertex colours where no frame observes it.  pose_rt:
        optional float32 [F, 12] (R row-major | t, world -> camera), else the engine's camera.  Returns a dict with image uint8 [H, W, 3]
        (R, G, B), uv float32 [F, 3, 2] (per face corner, v up as an OBJ reads it) and info (I3DTextureInfo).  Write it with
        mesh.save_textured_obj."""
        if pose_rt is not None:
            pose_rt = np.ascontiguousarray(pose_rt, np.float32)
            assert pose_rt.shape == (self.F, 12)
        prm = I3DTextureParams(int(texels_per_face), float(max_occlusion_distance), int(max_num_observations), 0)
        info = I3DTextureInfo()
        self._check(self.L.i3d_bake_texture(self.h, C.byref(prm), _p(pose_rt, C.c_float), C.byref(info)))
        out = dict(image=np.empty((info.atlas_height, info.atlas_width, 3), np.uint8), uv=np.empty((int(info.num_faces), 3, 2), np.float32), info=info)
        self._check(self.L.i3d_download_texture(self.h, _p(out["image"], C.c_uint8), _p(out["uv"], C.c_float)))
        return out

    def decompose_texture(self, min_shading: float = 0.05, sh=None):
        """Splits the texture of the resident mesh (the last bake_texture) into albedo and shading on the device (DESIGN.md §6x): at each
        owned texel's point and face normal, s = sh . basis(n) under sh (None: the subvolume SH of the last estimate_lighting; else nine
        coefficients used everywhere), and albedo = colour / 255 / s where the normal is not 0 and s > min_shading, else 0.  Returns a
        dict with albedo float32 [H, W, 3] (R, G, B), shading float32 [H, W] and info (I3DIntrinsicTextureInfo).  The albedo is known up
        to one global scale; mesh.albedo_image turns it into an image for mesh.save_textured_obj."""
        prm = I3DIntrinsicTextureParams(sh_lighting(sh), float(min_shading), 0)
        info = I3DIntrinsicTextureInfo()
        self._check(self.L.i3d_decompose_texture(self.h, C.byref(prm), C.byref(info)))
        H, W = info.atlas_height, info.atlas_width
        out = dict(albedo=np.empty((H, W, 3), np.float32), shading=np.empty((H, W), np.float32), info=info)
        self._check(self.L.i3d_download_intrinsic_texture(self.h, _p(out["albedo"], C.c_float), _p(out["shading"], C.c_float)))
        return out

    def set_relight(self, sh=None):
        """The lighting of rasterize_keyframes / rasterize_views with color="relit": None (default) for the subvolume SH of the lighting
        estimate at the time of the rasterization, else nine coefficients used everywhere."""
        self._check(self.L.i3d_set_relight(self.h, C.byref(sh_lighting(sh))))

    def upload_reference_mesh(self, mesh):
        """Uploads a reference surface for surface_distance: a dict with vertices float32 [V, 3] and faces int32 [F, 3] (an extract_mesh
        dict; its colours are ignored).  It replaces the previous reference and stays through grid, frame and mesh changes."""
        v = np.ascontiguousarray(mesh["vertices"], np.float32).reshape(-1, 3)
        f = np.ascontiguousarray(mesh["faces"], np.int32).reshape(-1, 3)
        self._check(self.L.i3d_upload_reference_mesh(self.h, len(v), _p(v, C.c_float), len(f), _p(f, C.c_int32)))

    def surface_distance(self, thresholds=(0.0002, 0.0005, 0.001), max_distance: float = 0.01, samples_per_edge: int = 2, cell_size=None):
        """Distances between the resident mesh (the last extract_mesh or simplify_mesh) and the reference mesh, on the device (DESIGN.md
        §6u).  Every face of either mesh is sampled at samples_per_edge^2 area-uniform points, and each point gets the nearest face of the
        other mesh within max_distance (metres).  Returns a dict with accuracy (resident -> reference) and completeness (reference ->
        resident), each with the sample counts, area, area-weighted mean / rms / max distance over the matched samples and the area
        fraction within each threshold; precision, recall and fscore per threshold; vertex_distance float32 [V] (inf beyond max_distance)
        and vertex_face int32 [V] (-1 then) of the resident mesh's vertices; and info (I3DDistanceInfo, with the grids and device times).
        cell_size None picks the search grid's cell edge automatically; the results do not depend on it."""
        thresholds = [float(t) for t in thresholds]
        if len(thresholds) > DISTANCE_MAX_THRESHOLDS:
            raise ValueError(f"at most {DISTANCE_MAX_THRESHOLDS} thresholds, got {len(thresholds)}")
        prm = I3DDistanceParams(int(samples_per_edge), float(max_distance), 0.0 if cell_size is None else float(cell_size), len(thresholds),
                                (C.c_float * DISTANCE_MAX_THRESHOLDS)(*thresholds))
        info = I3DDistanceInfo()
        self._check(self.L.i3d_surface_distance(self.h, C.byref(prm), C.byref(info)))
        V = int(info.num_vertices)
        vd, vf = np.empty(V, np.float32), np.empty(V, np.int32)
        self._check(self.L.i3d_download_surface_distance(self.h, _p(vd, C.c_float), _p(vf, C.c_int32)))
        nt = len(thresholds)

        def side(s):
            d = s.as_dict()
            d["fraction"] = d["fraction"][:nt]
            return d
        return dict(accuracy=side(info.side[0]), completeness=side(info.side[1]), thresholds=thresholds, precision=list(info.precision)[:nt],
                    recall=list(info.recall)[:nt], fscore=list(info.fscore)[:nt], vertex_distance=vd, vertex_face=vf, info=info)

    def debug_distance_samples(self, direction: int, n: int):
        """(d2 float32 [n], face int32 [n]) per sample of the last surface_distance after debug_set_keep_distance_samples(True); direction
        0 = resident -> reference, 1 = reference -> resident; n = that side's num_samples"""
        d2, face = np.empty(n, np.float32), np.empty(n, np.int32)
        self._check(self.L.i3d_debug_get_distance_samples(self.h, int(direction), _p(d2, C.c_float), _p(face, C.c_int32)))
        return d2, face

    def debug_set_keep_distance_samples(self, on: bool = True):
        self._check(self.L.i3d_debug_set_keep_distance_samples(self.h, 1 if on else 0))

    def register_reference_mesh(self, max_distance=(0.016, 0.008, 0.004), iterations=(10, 10, 10), samples_per_edge: int = 1,
                                min_normal_cos: float = 0.5, min_correspondences: int = 100, cell_size=None, init=None):
        """Estimates the rigid T that maps the reference mesh onto the resident mesh (x_resident = R x_reference + t), on the device
        (DESIGN.md §6aa): point-to-plane ICP of the resident mesh's area samples against the reference's faces, one stage per
        (max_distance metres, iterations) pair, coarse to fine, from init (T [12] R row-major | t; None = identity).  Returns (T float64
        [12], info I3DRegisterInfo).  Nothing else changes; transform_reference_mesh(T) moves the reference.  cell_size None picks the
        search grid's cell edge automatically; the result does not depend on it."""
        md, it = [float(d) for d in max_distance], [int(i) for i in iterations]
        if len(md) != len(it) or not 1 <= len(md) <= REGISTER_MAX_STAGES:
            raise ValueError(f"max_distance and iterations need the same length in [1, {REGISTER_MAX_STAGES}], got {len(md)} and {len(it)}")
        pad = REGISTER_MAX_STAGES - len(md)
        prm = I3DRegisterParams(int(samples_per_edge), len(md), (C.c_float * REGISTER_MAX_STAGES)(*(md + [0.0] * pad)),
                                (C.c_int32 * REGISTER_MAX_STAGES)(*(it + [0] * pad)), float(min_normal_cos), int(min_correspondences),
                                0.0 if cell_size is None else float(cell_size))
        T0 = None if init is None else np.ascontiguousarray(init, np.float64).reshape(12)
        T = np.empty(12, np.float64)
        info = I3DRegisterInfo()
        self._check(self.L.i3d_register_reference_mesh(self.h, C.byref(prm), _p(T0, C.c_double), _p(T, C.c_double), C.byref(info)))
        return T, info

    def transform_reference_mesh(self, T):
        """Moves the reference mesh by T [12] (R row-major | t) on the device: x <- float(R x + t), in double"""
        T = np.ascontiguousarray(T, np.float64).reshape(12)
        self._check(self.L.i3d_transform_reference_mesh(self.h, _p(T, C.c_double)))

    def debug_register_systems(self, num_samples: int):
        """The last register_reference_mesh's systems float64 [n, 31] (the 29 tracker sums, sum w for the first and the last system, 0),
        the pose T^-1 each was formed at float64 [n, 12], and the per-sample nearest face at the initial pose int32 [num_samples]"""
        n = C.c_int32()
        self._check(self.L.i3d_debug_get_register_systems(self.h, C.byref(n), None, None, None))
        S, M = np.empty((n.value, 31), np.float64), np.empty((n.value, 12), np.float64)
        f = np.empty(num_samples, np.int32)
        self._check(self.L.i3d_debug_get_register_systems(self.h, C.byref(n), _p(S, C.c_double), _p(M, C.c_double), _p(f, C.c_int32)))
        return S, M, f

    def grid_from_mesh(self, source: str = "reference", voxel_size: float = 0.002, band: float = 3.0, cell_size=None):
        """Replaces the voxel set by the narrow-band signed distance field of a triangle mesh, built on the device (DESIGN.md §6v): every
        voxel c (at c * voxel_size metres) with a face within band voxels gets sdf0 = sdf = the signed distance to the nearest face, signed
        by the angle-weighted pseudonormal of the closest feature, albedo 0.6, weight 1 and colour 0 (recompute_colors colours it).
        source "reference" converts the mesh of upload_reference_mesh (for example one read with mesh.load_ply), "resident" the last
        extract_mesh or simplify_mesh.  An open mesh gets no voxels past its rim.  cell_size None picks the search grid's cell edge
        automatically; the result does not depend on it.  The frames, camera and reference mesh stay; everything derived from the old
        voxel set (SH, lighting, mesh, texture, render) is dropped.  Returns (voxels, info), info an I3DGridFromMeshInfo with the counts
        and the device ms per stage."""
        if source not in GRID_FROM_MESH_SOURCES:
            raise ValueError(f"source must be one of {sorted(GRID_FROM_MESH_SOURCES)}, got {source!r}")
        prm = I3DGridFromMeshParams(GRID_FROM_MESH_SOURCES[source], float(voxel_size), float(band), 0.0 if cell_size is None else float(cell_size))
        info = I3DGridFromMeshInfo()
        self._check(self.L.i3d_grid_from_mesh(self.h, C.byref(prm), C.byref(info)))
        self.n = int(info.num_voxels)
        return self.n, info

    def debug_grid_from_mesh_voxels(self, n: int):
        """(face int32 [n], feature int8 [n]) per voxel of the last grid_from_mesh: the nearest face and the I3D_FEATURE_* of the closest
        point (0, 1, 2 vertex a, b, c; 3, 4, 5 edge ab, ac, bc; 6 interior)"""
        face, feat = np.empty(n, np.int32), np.empty(n, np.int8)
        self._check(self.L.i3d_debug_get_grid_from_mesh_voxels(self.h, _p(face, C.c_int32), _p(feat, C.c_int8)))
        return face, feat

    def mode_colors(self, mode: str, source: str = "refined"):
        """Every voxel's colour in colour mode `mode` (a mode string of extract_mesh), uint8 [n, 3] in the grid's order: the colours a
        mesh of that mode interpolates.  The geometric modes read the sdf of `source`."""
        src = self._mesh_source(source)
        m = self._color_mode(mode)
        n = int(self.L.i3d_num_voxels(self.h))
        rgb = np.empty((n, 3), np.uint8)
        self._check(self.L.i3d_mode_colors(self.h, src, m, _p(rgb, C.c_uint8)))
        return rgb

    # ---- rendering the surface into the keyframes (DESIGN.md §6m) -------------------------------------------------------------
    def render_keyframes(self, ids, source: str = "refined", planes=("depth", "normal", "albedo", "shading", "intensity"),
                         photometric: bool = True):
        """Ray-casts the zero level set of `source` ("fused": sdf0, "refined") into the frames `ids` with the engine's current camera,
        at the size of the installed frames.  Returns a dict with the requested planes, float32 [n, H, W] (normal [n, H, W, 3]), and
        stats: one dict per view (I3DRenderStats: hit / observed pixel counts, depth pairs and photometric pairs with their sums of
        |error| and error^2).  planes=() gives the statistics only.  photometric=False skips the shading and the photometric pairs, so
        no per-voxel SH is needed.  Device time: phase_ms("render")."""
        src = self._mesh_source(source)
        mask = 0
        for p in planes:
            if p not in RENDER_PLANES:
                raise ValueError(f"plane must be one of {sorted(RENDER_PLANES)}, got {p!r}")
            mask |= RENDER_PLANES[p]
        ids, n = self._ids(ids)
        prm = I3DRenderParams(src, mask, 1 if photometric else 0, 0)
        stats = (I3DRenderStats * max(n, 1))()
        self._check(self.L.i3d_render_keyframes(self.h, C.c_int32(n), _p(ids, C.c_int32), C.byref(prm), stats))
        W, H = self.frame_size
        out = {p: np.empty((n, H, W, 3) if p == "normal" else (n, H, W), np.float32) for p in RENDER_PLANES if RENDER_PLANES[p] & mask}
        if out:
            self._check(self.L.i3d_download_render(self.h, *(_p(out.get(p), C.c_float) for p in RENDER_PLANES)))
        out["stats"] = [stats[i].as_dict() for i in range(n)]
        return out

    def set_render_skip(self, on: bool):
        """True (default): the renderer jumps over empty 8^3 bricks; False: it evaluates every lattice sample (same results)."""
        self._check(self.L.i3d_debug_set_render_skip(self.h, C.c_int(1 if on else 0)))

    # ---- rasterizing the resident mesh into the keyframes and into new views (DESIGN.md §6w) ---------------------------------
    @staticmethod
    def _raster_params(color, planes):
        if color not in RASTER_COLORS:
            raise ValueError(f"color must be one of None, 'vertex', 'texture', 'relit', got {color!r}")
        mask = 0
        for p in planes:
            if p not in RASTER_PLANES:
                raise ValueError(f"plane must be one of {sorted(RASTER_PLANES)}, got {p!r}")
            mask |= RASTER_PLANES[p]
        return I3DRasterParams(mask, RASTER_COLORS[color])

    def _download_raster(self, n, W, H, mask):
        shapes = dict(depth=((n, H, W), np.float32), face=((n, H, W), np.int32), bary=((n, H, W, 2), np.float32),
                      normal=((n, H, W, 3), np.float32), rgb=((n, H, W, 3), np.uint8))
        ctype = dict(depth=C.c_float, face=C.c_int32, bary=C.c_float, normal=C.c_float, rgb=C.c_uint8)
        out = {p: np.empty(*shapes[p]) for p in RASTER_PLANES if RASTER_PLANES[p] & mask}
        if out:
            self._check(self.L.i3d_download_raster(self.h, *(_p(out.get(p), ctype[p]) for p in RASTER_PLANES)))
        return out

    def rasterize_keyframes(self, ids, color="vertex", planes=("depth", "face", "bary", "normal", "rgb")):
        """Rasterizes the resident mesh (the last extract_mesh or simplify_mesh) into the frames `ids` with the engine's current camera,
        at the size of the installed frames (DESIGN.md §6w).  color: "vertex" (the vertex colours), "texture" (the last bake_texture of
        the resident mesh), "relit" (the albedo of the last decompose_texture times the shading under set_relight's lighting, §6x) or
        None.  Returns a dict with the requested planes [n, H, W] (depth float32, 0 = no face; face int32, -1 = no
        face; bary float32 [.., 2]; normal float32 [.., 3], world frame; rgb uint8 [.., 3]), stats: one dict per view (I3DRasterStats:
        covered / observed pixels, depth pairs with sum |e| and e^2 in metres, colour pairs with per-channel integer sums of |e| and e^2
        against the colour frame) and info (I3DRasterInfo).  planes=() gives the statistics only."""
        prm = self._raster_params(color, planes)
        ids, n = self._ids(ids)
        stats = (I3DRasterStats * max(n, 1))()
        info = I3DRasterInfo()
        self._check(self.L.i3d_rasterize_keyframes(self.h, C.c_int32(n), _p(ids, C.c_int32), C.byref(prm), stats, C.byref(info)))
        W, H = self.frame_size
        out = self._download_raster(n, W, H, prm.planes)
        out["stats"] = [stats[i].as_dict() for i in range(n)]
        out["info"] = info
        return out

    def rasterize_views(self, camera: dict, poses, color="vertex", planes=("depth", "face", "bary", "normal", "rgb")):
        """Rasterizes the resident mesh into new views: camera a dict with fx, fy, cx, cy (pixels), width, height and optionally
        distortion (k1, k2, p1, p2, k3); poses float32 [n, 12] (R row-major | t, world -> camera).  Returns the planes of
        rasterize_keyframes and info; no statistics."""
        prm = self._raster_params(color, planes)
        poses = np.ascontiguousarray(poses, np.float32).reshape(-1, 12)
        n = int(poses.shape[0])
        d = [float(x) for x in camera.get("distortion", (0.0,) * 5)]
        cam = I3DRasterCamera(float(camera["fx"]), float(camera["fy"]), float(camera["cx"]), float(camera["cy"]), (C.c_float * 5)(*d),
                              int(camera["width"]), int(camera["height"]))
        info = I3DRasterInfo()
        self._check(self.L.i3d_rasterize_views(self.h, C.c_int32(n), C.byref(cam), _p(poses, C.c_float), C.byref(prm), C.byref(info)))
        out = self._download_raster(n, cam.width, cam.height, prm.planes)
        out["info"] = info
        return out

    def set_raster_binning(self, on: bool):
        """True (default): faces are binned to 8 x 8 pixel tiles; False: every face is tested against every pixel (same results)."""
        self._check(self.L.i3d_debug_set_raster_binning(self.h, C.c_int(1 if on else 0)))

    def set_raster_batch(self, views: int):
        """views > 0: rasterize in passes of at most that many views; 0: as large as memory for 2^27 keys allows (same results)."""
        self._check(self.L.i3d_debug_set_raster_batch(self.h, C.c_int(int(views))))

    # ---- keyframe selection and the RGB-D pyramid (KeyframeSelection::estimateBlur, Pyramid::create) ----------------------
    def keyframe_scores(self, bgr):
        """Blur score (Crete 2007, 1 = sharp) of every frame: bgr uint8 [F, H, W, 3] (B, G, R) -> float64 [F]; NaN for a frame without
        vertical variation.  Pick the keyframes with keyframes.select_keyframes."""
        bgr = np.ascontiguousarray(bgr, np.uint8)
        assert bgr.ndim == 4 and bgr.shape[3] == 3
        F, H, W = bgr.shape[:3]
        out = np.empty(F, np.float64)
        self._check(self.L.i3d_keyframe_scores(self.h, C.c_int32(F), C.c_int32(W), C.c_int32(H), _p(bgr, C.c_uint8), _p(out, C.c_double)))
        return out

    def upload_rgbd_frames(self, bgr, depth, lum=None):
        """Level-0 keyframes into the device frame store: bgr uint8 [F, H, W, 3], depth float32 [F, H, W] metres, lum float32 [F, H, W] or
        None (computed from bgr).  use_rgbd_level(l) then installs pyramid level l."""
        bgr = np.ascontiguousarray(bgr, np.uint8)
        depth = np.ascontiguousarray(depth, np.float32)
        F, H, W = depth.shape
        assert bgr.shape == (F, H, W, 3)
        if lum is not None:
            lum = np.ascontiguousarray(lum, np.float32)
            assert lum.shape == (F, H, W)
        self._check(self.L.i3d_upload_rgbd_frames(self.h, C.c_int32(F), C.c_int32(W), C.c_int32(H), _p(bgr, C.c_uint8), _p(depth, C.c_float),
                                                  _p(lum, C.c_float)))
        self._store_F = F

    def use_rgbd_level(self, lvl: int):
        """Builds pyramid level `lvl` of the stored keyframes on the device and makes it the engine's frames (as upload_frames would, at scale
        2^-lvl; at level 0 the colours too).  Returns (W, H) of the level."""
        w, h = C.c_int32(0), C.c_int32(0)
        self._check(self.L.i3d_use_rgbd_level(self.h, C.c_int32(int(lvl)), C.byref(w), C.byref(h)))
        self.F = self._store_F
        self.frame_size = (int(w.value), int(h.value))
        return self.frame_size

    # ---- the sensor store: the raw sequence on the device (Sensor::depth / Sensor::color) ------------------------------------
    def sensor_frames_begin(self, depth_cam, color_cam, capacity: int):
        """Starts an empty device store of `capacity` frames for a depth camera and a colour camera, each (W, H, fx, fy, cx, cy); its
        device memory is allocated here, so a long sequence can be added in chunks."""
        dc, cc = fusion_camera(depth_cam), fusion_camera(color_cam)
        self._check(self.L.i3d_sensor_frames_begin(self.h, C.byref(dc), C.byref(cc), C.c_int32(int(capacity))))
        self._sensor_cams = (dc, cc)

    def sensor_frames_add(self, depth, bgr):
        """Appends frames: depth float32 [F, Hd, Wd] metres (range-thresholded), bgr uint8 [F, Hc, Wc, 3] (B, G, R)."""
        dc, cc = self._sensor_cams
        depth = np.ascontiguousarray(depth, np.float32)
        bgr = np.ascontiguousarray(bgr, np.uint8)
        F = int(depth.shape[0])
        assert depth.shape == (F, dc.height, dc.width) and bgr.shape == (F, cc.height, cc.width, 3)
        self._check(self.L.i3d_sensor_frames_add(self.h, C.c_int32(F), _p(depth, C.c_float), _p(bgr, C.c_uint8)))

    def sensor_num_frames(self) -> int:
        return int(self.L.i3d_sensor_num_frames(self.h))

    def sensor_keyframe_scores(self):
        """keyframe_scores of every stored frame, read from the store: float64 [sensor_num_frames()]."""
        out = np.empty(self.sensor_num_frames(), np.float64)
        self._check(self.L.i3d_sensor_keyframe_scores(self.h, _p(out, C.c_double)))
        return out

    @staticmethod
    def _ids(ids):
        ids = np.ascontiguousarray(ids, np.int32).ravel()
        return ids, int(ids.shape[0])

    def fusion_integrate_sensor(self, ids, pose_cam_to_world, pose_world_to_cam):
        """fusion_integrate of the stored frames `ids`, in list order; poses float32 [len(ids), 12] (R row-major | t)."""
        ids, n = self._ids(ids)
        c2w = np.ascontiguousarray(pose_cam_to_world, np.float32)
        w2c = np.ascontiguousarray(pose_world_to_cam, np.float32)
        assert c2w.shape == (n, 12) and w2c.shape == (n, 12)
        self._check(self.L.i3d_fusion_integrate_sensor(self.h, C.c_int32(n), _p(ids, C.c_int32), _p(c2w, C.c_float), _p(w2c, C.c_float)))

    # ---- tracking stored frames against the surface (DESIGN.md §6n) --------------------------------------------------------------
    @staticmethod
    def _track_params(sdf_source, params):
        p = default_track_params()
        p.sdf_source = sdf_source
        for k, v in params.items():
            if k == "iterations":
                v = list(v) + [0] * (TRACK_LEVELS - len(v))
                if len(v) != TRACK_LEVELS:
                    raise ValueError(f"iterations takes at most {TRACK_LEVELS} values")
                for i, x in enumerate(v):
                    p.iterations[i] = int(x)
            elif k in ("num_levels", "min_correspondences"):
                setattr(p, k, int(v))
            elif k in ("max_distance", "min_normal_cos"):
                setattr(p, k, float(v))
            else:
                raise ValueError(f"unknown tracking parameter {k!r}")
        return p

    @staticmethod
    def _track_color_params(color, ref=False):
        """I3DTrackColorParams from a dict: weight (one value for every level, or up to 4 values, level 0 first), max_color_diff,
        min_color_gradient, norm_radius, norm_eps; the rest keep default_track_color_params() (ref: default_track_color_ref_params(), or
        default_track_color_lni_params() when norm_radius > 0)."""
        color = color or {}
        if ref:
            p = default_track_color_lni_params() if int(color.get("norm_radius", 0)) > 0 else default_track_color_ref_params()
        else:
            p = default_track_color_params()
        for k, v in color.items():
            if k == "weight":
                v = [float(v)] * TRACK_LEVELS if np.ndim(v) == 0 else list(v) + [0.0] * (TRACK_LEVELS - len(v))
                if len(v) != TRACK_LEVELS:
                    raise ValueError(f"weight takes at most {TRACK_LEVELS} values")
                for i, x in enumerate(v):
                    p.weight[i] = float(x)
            elif k in ("max_color_diff", "min_color_gradient", "norm_eps"):
                setattr(p, k, float(v))
            elif k == "norm_radius":
                p.norm_radius = int(v)
            else:
                raise ValueError(f"unknown colour tracking parameter {k!r}")
        return p

    def _track_call(self, fn, ids, pose, name, n_pose, p, color=None, ref=None):
        """ref: (ref_ids, ref_pose) of a _ref call, passed after the pose"""
        ids, n = self._ids(ids)
        if pose is not None:
            pose = np.ascontiguousarray(pose, np.float64)
            if pose.shape != (n_pose(n), 12):
                raise ValueError(f"{name} must be [{n_pose(n)}, 12], got {pose.shape}")
        refs = ()
        if ref is not None:
            rid = np.ascontiguousarray(ref[0], np.int32).reshape(-1)
            rpose = np.ascontiguousarray(ref[1], np.float64)
            if rid.shape != (n,) or rpose.shape != (n, 12):
                raise ValueError(f"ref_ids and ref_pose_w2c must be [{n}] and [{n}, 12], got {rid.shape} and {rpose.shape}")
            refs = (_p(rid, C.c_int32), _p(rpose, C.c_double))
        out = np.empty((max(n, 1), 12), np.float64)
        infos = (I3DTrackInfo * max(n, 1))()
        if color is None:
            self._check(fn(self.h, C.c_int32(n), _p(ids, C.c_int32), _p(pose, C.c_double), C.byref(p), _p(out, C.c_double), infos))
            return out[:n], [infos[i].as_dict() for i in range(n)]
        cinfos = (I3DTrackColorInfo * max(n, 1))()
        self._check(fn(self.h, C.c_int32(n), _p(ids, C.c_int32), _p(pose, C.c_double), *refs, C.byref(p), C.byref(color), _p(out, C.c_double),
                       infos, cinfos))
        return out[:n], [dict(infos[i].as_dict(), color=cinfos[i].as_dict()) for i in range(n)]

    def track_sensor_frames(self, ids, pose_w2c, source: str = "fused", **params):
        """Point-to-plane ICP of the stored frames `ids` (distinct) against the surface of `source` ("fused": sdf0, "refined"), over the
        depth pyramid, starting from pose_w2c float64 [len(ids), 12] (world -> camera, R row-major | t).  params: fields of
        I3DTrackParams (num_levels, iterations (up to 4 values, level 0 first), max_distance, min_normal_cos, min_correspondences);
        the rest keep default_track_params().  Returns (poses float64 [n, 12] world -> camera, infos: one dict per frame).
        Device time: phase_ms("track")."""
        p = self._track_params(self._mesh_source(source), params)
        return self._track_call(self.L.i3d_track_sensor_frames, ids, pose_w2c, "pose_w2c", lambda n: n, p)

    # ---- tracking against the fusion in progress, and RGB-D odometry (DESIGN.md §6o) ---------------------------------------------
    def fusion_track_sensor_frames(self, ids, pose_w2c, **params):
        """track_sensor_frames with the fusion volume in progress as the model (equal to fusion_finish with correct_sdf_iterations 0
        followed by track_sensor_frames(..., "fused"), but the fusion goes on).  Returns (poses float64 [n, 12], infos)."""
        p = self._track_params(0, params)
        return self._track_call(self.L.i3d_fusion_track_sensor_frames, ids, pose_w2c, "pose_w2c", lambda n: n, p)

    def fusion_track_and_integrate_sensor(self, ids, pose_first=None, **params):
        """Dense odometry: each stored frame of `ids` (in order, repeats allowed) is tracked against the fusion in progress from a
        constant-velocity guess and integrated at the tracked pose; pose_first (world -> camera [12]) is the guess of the first frame,
        None continues from the previous call.  A frame that fails to track is not integrated.  Returns (poses float64 [n, 12] world ->
        camera, infos with status "anchored" (4) for a frame integrated untracked into an empty volume).  Time: phase_ms("odometry")."""
        p = self._track_params(0, params)
        pose = None if pose_first is None else np.asarray(pose_first, np.float64).reshape(1, 12)
        return self._track_call(self.L.i3d_fusion_track_and_integrate_sensor, ids, pose, "pose_first", lambda n: 1, p)

    # ---- tracking with colour as well as depth (DESIGN.md §6p) ------------------------------------------------------------------
    def track_sensor_frames_rgbd(self, ids, pose_w2c, source: str = "fused", color=None, **params):
        """track_sensor_frames with the photometric term: color = dict of I3DTrackColorParams fields (weight: lambda for every level
        or up to 4 values, level 0 first; max_color_diff; min_color_gradient), the rest default_track_color_params().  Returns
        (poses, infos); each info also has "color": the photometric rows and sum r^2 of the first and the last evaluated system."""
        p = self._track_params(self._mesh_source(source), params)
        return self._track_call(self.L.i3d_track_sensor_frames_rgbd, ids, pose_w2c, "pose_w2c", lambda n: n, p, self._track_color_params(color))

    def fusion_track_sensor_frames_rgbd(self, ids, pose_w2c, color=None, **params):
        """fusion_track_sensor_frames with the photometric term (see track_sensor_frames_rgbd)."""
        p = self._track_params(0, params)
        return self._track_call(self.L.i3d_fusion_track_sensor_frames_rgbd, ids, pose_w2c, "pose_w2c", lambda n: n, p,
                                self._track_color_params(color))

    def fusion_track_and_integrate_sensor_rgbd(self, ids, pose_first=None, color=None, **params):
        """fusion_track_and_integrate_sensor (dense odometry) with the photometric term (see track_sensor_frames_rgbd)."""
        p = self._track_params(0, params)
        pose = None if pose_first is None else np.asarray(pose_first, np.float64).reshape(1, 12)
        return self._track_call(self.L.i3d_fusion_track_and_integrate_sensor_rgbd, ids, pose, "pose_first", lambda n: 1, p,
                                self._track_color_params(color))

    # ---- the photometric term against a reference frame's image (DESIGN.md §6q) ----------------------------------------------------
    def track_sensor_frames_rgbd_ref(self, ids, pose_w2c, ref_ids, ref_pose_w2c, source: str = "fused", color=None, **params):
        """track_sensor_frames_rgbd with the model intensity of frame k sampled from the stored frame ref_ids[k] (may be ids[k] itself) at
        its world -> camera pose ref_pose_w2c[k] float64 [12] instead of from the voxel colours.  Returns (poses, infos) as the _rgbd call.
        color=dict(norm_radius=r, norm_eps=eps) with r > 0 compares locally normalised intensity (DESIGN.md §6r); the colour parameters
        not given then keep default_track_color_lni_params(), in normalised units."""
        p = self._track_params(self._mesh_source(source), params)
        return self._track_call(self.L.i3d_track_sensor_frames_rgbd_ref, ids, pose_w2c, "pose_w2c", lambda n: n, p,
                                self._track_color_params(color, True), ref=(ref_ids, ref_pose_w2c))

    def fusion_track_sensor_frames_rgbd_ref(self, ids, pose_w2c, ref_ids, ref_pose_w2c, color=None, **params):
        """fusion_track_sensor_frames_rgbd with the reference model (see track_sensor_frames_rgbd_ref)."""
        p = self._track_params(0, params)
        return self._track_call(self.L.i3d_fusion_track_sensor_frames_rgbd_ref, ids, pose_w2c, "pose_w2c", lambda n: n, p,
                                self._track_color_params(color, True), ref=(ref_ids, ref_pose_w2c))

    def fusion_track_and_integrate_sensor_rgbd_ref(self, ids, pose_first=None, color=None, **params):
        """Dense odometry with the reference model: each frame's reference is the last frame the loop integrated, at the pose it was
        integrated with; a frame without one (the first after pose_first, a fusion_begin or an integrate) is tracked on depth alone."""
        p = self._track_params(0, params)
        pose = None if pose_first is None else np.asarray(pose_first, np.float64).reshape(1, 12)
        return self._track_call(self.L.i3d_fusion_track_and_integrate_sensor_rgbd_ref, ids, pose, "pose_first", lambda n: 1, p,
                                self._track_color_params(color, True))

    def debug_track_reference_planes(self, level, n):
        """The last pass's planes of the last _ref call (`n` = its frame count) at pyramid `level`, each [n, H_l, W_l]: model (NaN where
        there is no model value), ref_intensity and ref_depth.  With norm_radius > 0 the model and ref_intensity are the normalised
        values the rows read (DESIGN.md §6r)."""
        dc = self._sensor_cams[0]
        Wl, Hl = dc.width, dc.height
        for _ in range(level):
            Wl, Hl = Wl // 2, Hl // 2
        out = {k: np.empty((n, Hl, Wl), np.float32) for k in ("model", "ref_intensity", "ref_depth")}
        m = C.c_int32(0)
        self._check(self.L.i3d_debug_get_track_reference_planes(self.h, C.c_int32(int(level)), _p(out["model"], C.c_float),
                                                                _p(out["ref_intensity"], C.c_float), _p(out["ref_depth"], C.c_float), C.byref(m)))
        assert m.value == n, (m.value, n)
        return out

    def debug_track_color_system(self, n):
        """the unweighted photometric sums float64 [n, 29] of the last evaluated system of each frame of the last _rgbd call of n frames"""
        sums = np.empty((n, 29), np.float64)
        self._check(self.L.i3d_debug_get_track_color_system(self.h, _p(sums, C.c_double)))
        return sums

    def debug_track_color_planes(self, level, frames, model_intensity=True):
        """The last pass's colour planes of the last _rgbd call (`frames` = its frame count): model_intensity [frames, H, W] and the
        frame intensity / grad_x / grad_y at pyramid `level`.  model_intensity=False leaves the model plane out (None), as after a _ref
        call, whose model planes debug_track_reference_planes returns.  After a _ref call with norm_radius > 0 the intensity (and the
        gradients of it) is the normalised plane the rows read (DESIGN.md §6r)."""
        dc = self._sensor_cams[0]
        W, H = dc.width, dc.height
        Wl, Hl = W, H
        for _ in range(level):
            Wl, Hl = Wl // 2, Hl // 2
        out = dict(model_intensity=np.empty((frames, H, W), np.float32) if model_intensity else None,
                   intensity=np.empty((frames, Hl, Wl), np.float32),
                   grad_x=np.empty((frames, Hl, Wl), np.float32), grad_y=np.empty((frames, Hl, Wl), np.float32))
        m = C.c_int32(0)
        self._check(self.L.i3d_debug_get_track_color_planes(self.h, C.c_int32(int(level)), _p(out["model_intensity"], C.c_float),
                                                            _p(out["intensity"], C.c_float), _p(out["grad_x"], C.c_float),
                                                            _p(out["grad_y"], C.c_float), C.byref(m)))
        assert m.value == frames, (m.value, frames)
        return out

    def debug_track_system(self, n):
        """(sums float64 [n, 29], pose camera -> world float64 [n, 12]) of the last tracking call of n frames."""
        sums, pose = np.empty((n, 29), np.float64), np.empty((n, 12), np.float64)
        self._check(self.L.i3d_debug_get_track_system(self.h, _p(sums, C.c_double), _p(pose, C.c_double)))
        return sums, pose

    def debug_track_planes(self, level, frames):
        """The last pass's planes of the last tracking call (`frames` = its frame count): dict of depth / normal at pyramid `level`,
        pred_depth / pred_normal of the prediction and the level-0 correspondence mask."""
        dc = self._sensor_cams[0]
        W, H = dc.width, dc.height
        Wl, Hl = W, H
        for _ in range(level):
            Wl, Hl = Wl // 2, Hl // 2
        out = dict(depth=np.empty((frames, Hl, Wl), np.float32), normal=np.empty((frames, Hl, Wl, 3), np.float32),
                   pred_depth=np.empty((frames, H, W), np.float32), pred_normal=np.empty((frames, H, W, 3), np.float32),
                   mask=np.empty((frames, H, W), np.uint8))
        m = C.c_int32(0)
        self._check(self.L.i3d_debug_get_track_planes(self.h, C.c_int32(int(level)), _p(out["depth"], C.c_float), _p(out["normal"], C.c_float),
                                                      _p(out["pred_depth"], C.c_float), _p(out["pred_normal"], C.c_float),
                                                      _p(out["mask"], C.c_uint8), C.byref(m)))
        assert m.value == frames, (m.value, frames)
        return out

    def select_rgbd_frames(self, ids):
        """The stored frames `ids` (any order, repeats allowed) become the level-0 keyframes of the frame store, their depth resized to the
        colour camera (resizeDepth), as upload_rgbd_frames would make them; use_rgbd_level(l) then installs level l."""
        ids, n = self._ids(ids)
        self._check(self.L.i3d_select_rgbd_frames(self.h, C.c_int32(n), _p(ids, C.c_int32)))
        self._store_F = n

    def debug_frames(self, with_color=False):
        """(lum, depth, bgr or None) of the current level as the device holds them."""
        W, H = self.frame_size
        lum, depth = np.empty((self.F, H, W), np.float32), np.empty((self.F, H, W), np.float32)
        bgr = np.empty((self.F, H, W, 3), np.uint8) if with_color else None
        self._check(self.L.i3d_debug_get_frames(self.h, _p(lum, C.c_float), _p(depth, C.c_float), _p(bgr, C.c_uint8)))
        return lum, depth, bgr

    def download_state(self):
        sdf = np.empty(self.n, np.float64)
        alb = np.empty(self.n, np.float64)
        poses = np.empty((self.F, 6), np.float64)
        intr = np.empty(4, np.float64)
        dist = np.empty(5, np.float64)
        self._check(self.L.i3d_download_state(self.h, _p(sdf, C.c_double), _p(alb, C.c_double), _p(poses, C.c_double),
                                              _p(intr, C.c_double), _p(dist, C.c_double)))
        return dict(sdf_refined=sdf, albedo=alb, poses=poses, intr=intr, dist=dist)

    # ---- measurement / parity hooks ---------------------------------------------------------
    def phase_ms(self, name: str) -> float:
        return float(self.L.i3d_phase_ms(self.h, name.encode()))

    def phase_count(self, name: str) -> int:
        return int(self.L.i3d_phase_count(self.h, name.encode()))

    def set_kernel_timers(self, level: int):
        """0 (default): phases + the roofline kernels (first k_eg_apply of each solve); 1: every kernel of the iteration."""
        self.L.i3d_debug_set_kernel_timers(self.h, C.c_int(int(level)))

    def debug_rows(self, want_jac=True):
        S = int(self.L.i3d_debug_num_slots(self.h))
        voxel = np.empty(S, np.int32)
        frame = np.empty(S, np.int32)
        res = np.empty(S, np.float64)
        w = np.empty(S, np.float64)
        J = np.empty((29, S), np.float32) if want_jac else None
        self._check(self.L.i3d_debug_get_rows(self.h, _p(voxel, C.c_int32), _p(frame, C.c_int32), _p(res, C.c_double), _p(w, C.c_double),
                                              _p(J, C.c_float)))
        return dict(voxel=voxel, frame=frame, residual=res, raw_weight=w, J=J)

    def debug_observations(self, K: int):
        fr = np.empty((self.n, K), np.int32)
        w = np.empty((self.n, K), np.float32)
        act = np.empty(self.n, np.uint8)
        self._check(self.L.i3d_debug_get_observations(self.h, C.c_int32(K), _p(fr, C.c_int32), _p(w, C.c_float), _p(act, C.c_uint8)))
        return fr, w, act

    def debug_step(self):
        U = 2 * self.n + 6 * self.F + 9
        st = np.zeros(U, np.float64)
        fm = np.zeros(U, np.uint8)
        cs = np.zeros(U, np.float64)
        self._check(self.L.i3d_debug_get_step(self.h, _p(st, C.c_double), _p(fm, C.c_uint8), _p(cs, C.c_double)))
        return st, fm, cs

    def debug_pcg_vectors(self):
        """(x, p): the PCG iterate and search direction (float32 [U], Jacobi-scaled) as the last LM trial's solve left them."""
        U = 2 * self.n + 6 * self.F + 9
        x, p = np.empty(U, np.float32), np.empty(U, np.float32)
        self._check(self.L.i3d_debug_get_pcg_vectors(self.h, _p(x, C.c_float), _p(p, C.c_float)))
        return x, p

    def debug_normal_equations(self):
        """b = J'^T f, Jacobi scale s, jtj = s^2 colnorm^2 (float32 [U]) and the raw E_g camera sums cam_acc (float32 [33F + 43])."""
        U = 2 * self.n + 6 * self.F + 9
        b, s, jtj = np.empty(U, np.float32), np.empty(U, np.float32), np.empty(U, np.float32)
        cam = np.empty(33 * self.F + 43, np.float32)
        self._check(self.L.i3d_debug_get_normal_equations(self.h, _p(b, C.c_float), _p(s, C.c_float), _p(jtj, C.c_float), _p(cam, C.c_float)))
        return dict(b=b, s=s, jtj=jtj, cam_acc=cam)

    def debug_apply_operator(self, v):
        """q = S (J^T W J) S v for the rows of the last iteration (float32 [U]), through the production operator kernels."""
        U = 2 * self.n + 6 * self.F + 9
        v = np.ascontiguousarray(v, np.float32)
        assert v.shape == (U,)
        q = np.empty(U, np.float32)
        self._check(self.L.i3d_debug_apply_operator(self.h, _p(v, C.c_float), _p(q, C.c_float)))
        return q


def shard_range(n: int, rank: int, world: int, align: int = 512):
    """Voxel index range [begin, end) whose residual rows `rank` owns: equal contiguous ranges of the grid's
    iteration order (8^3-brick-major => z-slabs of bricks), aligned to whole bricks where possible."""
    if world <= 1:
        return 0, n
    per = -(-n // world)
    per = -(-per // align) * align
    b = min(n, rank * per)
    e = min(n, (rank + 1) * per)
    if rank == world - 1:
        e = n
    return b, e


def cut_ranges(cost, world: int, align: int = 64):
    """Cuts the index range [0, n) of a per-voxel cost vector (torch tensor, any device) into `world` contiguous ranges of (nearly) equal
    summed cost; every interior cut is rounded to a multiple of `align` voxels and the cuts are monotone.  Pure function of its input:
    every rank that passes the same (all-reduced) cost vector gets the same ranges."""
    import torch
    n = int(cost.shape[0])
    c = torch.cumsum(cost.to(torch.float64), 0)
    total = float(c[-1].item()) if n > 0 else 0.0
    cuts = [0]
    for r in range(1, world):
        i = int(torch.searchsorted(c, torch.tensor([total * r / world], device=c.device, dtype=c.dtype)).item())
        i = min(n, max(cuts[-1], (i + align // 2) // align * align))
        cuts.append(i)
    cuts.append(n)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def balanced_shard_ranges(eng, dist, params, n: int, align: int = 64, voxel_weight: float = 2.0):
    """Voxel index ranges [begin, end) per rank that balance the WORK rather than the voxel count: one residual build with the
    equal-count split (shard_range) gives, per voxel, the number of valid E_g rows; the cost model rows + voxel_weight * active is
    summed over ranks and cut into `world` equal parts (aligned to `align` voxels).  Call once per grid; returns a list of
    (begin, end) identical on every rank.  (z-slabs of a closed surface see very different numbers of frames: the equal-count
    split left the slowest rank with 1.7x the mean k_eg_apply time at 8 GPUs, profiles/r01 scaling table.)"""
    import torch
    world = dist.get_world_size()
    rank = dist.get_rank()
    eng.set_shard(*shard_range(n, rank, world))
    p = type(params).from_buffer_copy(bytes(params))
    p.build_only = 1
    eng.gn_iteration(p)
    rows = eng.debug_rows(want_jac=False)
    K = int(p.num_observations)
    stride = len(rows["frame"]) // max(K, 1)
    cost = np.zeros(n, np.float64)
    vox = rows["voxel"][:stride]
    valid = (rows["frame"].reshape(K, stride) >= 0).sum(0)
    m = vox >= 0
    cost[vox[m]] = valid[m] + voxel_weight
    t = torch.from_numpy(cost).cuda()
    dist.all_reduce(t)
    ranges = cut_ranges(t, world, align)
    if os.environ.get("I3D_SHARD", "balanced") != "timed":
        return ranges
    return rebalance_by_time(eng, dist, params, n, ranges, t, align)


TIMED_KERNELS = ("k_select_obs", "k_eg_build", "k_eg_accum", "k_eg_cost", "k_eg_apply", "k_op_partial", "k_cg_update", "k_cg_dir")


def rebalance_by_time(eng, dist, params, n, ranges, cost, align=64, rounds=2):
    """Second stage of the shard balance (I3D_SHARD=timed): the row-count model misses per-voxel differences the kernels see (the
    observation selection visits more frames for some slabs of a closed surface than for others).  One full GN iteration per round is
    timed per kernel on every rank (compute kernels only: the exchange kernels contain the waiting for the slowest rank), the model
    cost of every voxel is scaled by (measured time / model cost) of the rank that ran it, and the ranges are cut again.  The engine
    state is restored afterwards.  `cost`: the summed model cost per voxel (device tensor)."""
    import torch
    world, rank = dist.get_world_size(), dist.get_rank()
    saved = eng.download_state()
    p = type(params).from_buffer_copy(bytes(params))
    cost = cost.clone()
    for _ in range(rounds):
        eng.set_shard(*ranges[rank])
        eng.set_kernel_timers(1)
        eng.gn_iteration(p)                      # warm-up (launch attributes, first-touch)
        eng.upload_voxel_params(saved["sdf_refined"], saved["albedo"]); eng.set_camera(saved["poses"], saved["intr"], saved["dist"])
        eng.gn_iteration(p)
        mine = sum(eng.phase_ms(k) for k in TIMED_KERNELS)
        eng.set_kernel_timers(0)
        eng.upload_voxel_params(saved["sdf_refined"], saved["albedo"]); eng.set_camera(saved["poses"], saved["intr"], saved["dist"])
        tt = torch.zeros(world, device="cuda", dtype=torch.float64)
        tt[rank] = mine
        dist.all_reduce(tt)
        c = torch.cumsum(cost, 0)
        scale = torch.ones(world, device="cuda", dtype=torch.float64)
        for r, (b, e_) in enumerate(ranges):
            model = float((c[e_ - 1] - (c[b - 1] if b > 0 else 0.0)).item()) if e_ > b else 0.0
            if model > 0.0 and float(tt[r].item()) > 0.0:
                scale[r] = tt[r] / model
        for r, (b, e_) in enumerate(ranges):
            cost[b:e_] *= scale[r]
        ranges = cut_ranges(cost, world, align)
    return ranges


def _comm_init(self, rank: int, world: int, dist=None):
    """Creates the engine's NCCL communicator.  The 128-byte unique id is produced on rank 0 by the library and
    distributed with torch.distributed (`dist`, already initialised)."""
    if world <= 1:
        return
    import torch
    buf = (C.c_uint8 * 128)()
    if rank == 0:
        if self.L.i3d_comm_unique_id(buf) != 0:
            raise RuntimeError("i3d_comm_unique_id failed: " + self.L.i3d_last_error(None).decode())
    dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
    t = torch.tensor(list(buf), dtype=torch.uint8, device=dev)
    dist.broadcast(t, 0)
    raw = bytes(t.cpu().tolist())
    arr = (C.c_uint8 * 128).from_buffer_copy(raw)
    self._check(self.L.i3d_comm_init(self.h, C.c_int32(rank), C.c_int32(world), arr))
    self.rank, self.world = rank, world
    # peer-memory exchange: every rank maps every peer's mailbox (CUDA IPC).  I3D_XCHG=nccl keeps the ncclAllReduce path.
    self.p2p = False
    if os.environ.get("I3D_XCHG", "p2p") != "nccl" and dist.get_backend() == "nccl":
        mine = (C.c_uint8 * 64)()
        self._check(self.L.i3d_comm_p2p_export(self.h, mine))
        t = torch.tensor(list(mine), dtype=torch.uint8, device="cuda")
        allh = torch.empty(64 * world, dtype=torch.uint8, device="cuda")
        dist.all_gather_into_tensor(allh, t)
        rawh = bytes(allh.cpu().tolist())
        harr = (C.c_uint8 * (64 * world)).from_buffer_copy(rawh)
        rc = self.L.i3d_comm_p2p_connect(self.h, harr)
        ok = torch.tensor([1 if rc == 0 else 0], device="cuda")
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if ok.item() != 1:
            raise RuntimeError("i3d_comm_p2p_connect failed on some rank (" + self.L.i3d_last_error(self.h).decode() + "); set I3D_XCHG=nccl to use ncclAllReduce")
        self.p2p = True


def _set_shard(self, begin: int, end: int):
    self._check(self.L.i3d_set_shard(self.h, C.c_int64(begin), C.c_int64(end)))


Engine.comm_init = _comm_init
Engine.set_shard = _set_shard
