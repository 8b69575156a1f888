"""ctypes bindings of the C ABI declared in include/surfel_b200.h.

The same signatures are exported twice:
  * libsurfel_b200.so   (prefix `sm_`)    -- the product: hand-written sm_90a kernels
  * oracle/_ref/libsurfel_ref.so (prefix `smref_`) -- TEST INFRASTRUCTURE: the reference's
    own kernels rebuilt for sm_90a behind the same ABI. Only tests/, __graft_entry__.smoke()
    and bench.py's reference arm load it (see `load_reference_oracle`).

There is no CPU fallback: if the product library is missing or cannot be loaded the
import of the kernels fails loudly.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
REPO_ROOT = PKG_DIR.parent
LIB_PATH = PKG_DIR / "libsurfel_b200.so"
REF_LIB_PATH = REPO_ROOT / "oracle" / "_ref" / "libsurfel_ref.so"
# TEST INFRASTRUCTURE: the reference's restated host glue linked against the vis:: link shims
# (include/vis_shims/) instead of the reference's cuda_depth_processing.cu object.
SHIM_LIB_PATH = REPO_ROOT / "oracle" / "_ref" / "libsurfel_shimref.so"

SM_OK = 0
SM_ERR_CUDA = -1
SM_ERR_INVALID_ARGUMENT = -2
SM_ERR_CAPACITY = -3
INVALID_SURFEL_INDEX = 0xFFFFFFFF
ROW_COUNT = 25


class IntegrateParams(C.Structure):
    """sm_integrate_params; defaults = APP/main.cc:279-371."""
    _fields_ = [
        ("depth_scaling", C.c_float),
        ("sensor_noise_factor", C.c_float),
        ("max_surfel_confidence", C.c_float),
        ("regularizer_weight", C.c_float),
        ("regularization_frame_window_size", C.c_int32),
        ("do_blending", C.c_int32),
        ("measurement_blending_radius", C.c_int32),
        ("regularization_iterations_per_integration_iteration", C.c_int32),
        ("radius_factor_for_regularization_neighbors", C.c_float),
        ("normal_compatibility_threshold_deg", C.c_float),
        ("surfel_integration_active_window_size", C.c_int32),
    ]

    @classmethod
    def defaults(cls) -> "IntegrateParams":
        return cls(5000.0, 0.05, 5.0, 10.0, 30, 1, 12, 1, 2.0, 40.0, 2**31 - 1)


class PreprocessParams(C.Structure):
    """sm_preprocess_params; defaults = APP/main.cc:415-478."""
    _fields_ = [
        ("depth_scaling", C.c_float),
        ("max_depth", C.c_float),
        ("depth_valid_region_radius", C.c_float),
        ("bilateral_filter_sigma_xy", C.c_float),
        ("bilateral_filter_radius_factor", C.c_float),
        ("bilateral_filter_sigma_depth_factor", C.c_float),
        ("outlier_filtering_frame_count", C.c_int32),
        ("outlier_filtering_required_inliers", C.c_int32),
        ("outlier_filtering_depth_tolerance_factor", C.c_float),
        ("depth_erosion_radius", C.c_int32),
        ("observation_angle_threshold_deg", C.c_float),
        ("point_radius_extension_factor", C.c_float),
        ("point_radius_clamp_factor", C.c_float),
    ]

    @classmethod
    def defaults(cls) -> "PreprocessParams":
        return cls(5000.0, 3.0, 333.0, 3.0, 2.0, 0.05, 8, -1, 0.02, 2, 85.0, 1.5, float("inf"))


class StreamDesc(C.Structure):
    _fields_ = [
        ("width", C.c_int32), ("height", C.c_int32), ("frame_count", C.c_int32),
        ("frames_on_host", C.c_int32),
        ("depth", C.c_void_p), ("color", C.c_void_p),
        ("global_T_frame", C.c_void_p), ("frame_T_global", C.c_void_p),
        ("others_TR_reference", C.c_void_p),
    ]


class TransferToken(C.Structure):
    """sm_transfer_token: identifies the transfer that last filled a set of CUDASurfelBuffersCPU arrays."""
    _fields_ = [("generation", C.c_uint64), ("epoch", C.c_uint64), ("surfel_count", C.c_uint64)]


class TransferStats(C.Structure):
    _fields_ = [("surfel_count", C.c_uint64), ("changed_count", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("full_transfer", C.c_int32), ("reserved", C.c_int32)]


class VisualizationParams(C.Structure):
    """sm_visualization_params (arguments of UpdateVisualizationBuffers, cuda_surfel_reconstruction.cc:361-403)."""
    _fields_ = [("frame_index", C.c_uint32), ("latest_triangulated_frame_index", C.c_uint32),
                ("latest_mesh_surfel_count", C.c_uint32), ("surfel_integration_active_window_size", C.c_int32),
                ("point_size_in_floats", C.c_uint32), ("visualize_last_update_timestamp", C.c_int32),
                ("visualize_creation_timestamp", C.c_int32), ("visualize_radii", C.c_int32),
                ("visualize_normals", C.c_int32)]


class StreamStats(C.Structure):
    _fields_ = [
        ("frames_integrated", C.c_uint32), ("surfels_size", C.c_uint32), ("surfel_count", C.c_uint32),
        ("kernel_launches", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
        ("host_enqueue_ms", C.c_double),
    ]


class SessionStatus(C.Structure):
    """sm_session_status: progress of an incremental session after a push."""
    _fields_ = [("frames_pushed", C.c_uint32), ("frames_integrated", C.c_uint32),
                ("last_integrated_frame", C.c_int64)]


class RenderParams(C.Structure):
    """sm_render_params: output size, pinhole intrinsics (pixel-corner convention) and the depth range drawn."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fx", C.c_float), ("fy", C.c_float),
                ("cx", C.c_float), ("cy", C.c_float), ("near_depth", C.c_float), ("far_depth", C.c_float)]


RENDER_UNMESHED_SURFELS = 1
DISK_INDEX_FLAG = 0x80000000   # sm_render_mesh: the index of a pixel drawn by a disk

TRACK_CLOUD = 0
TRACK_PREVIOUS_FRAME = 1


class TrackParams(C.Structure):
    """sm_track_params: pyramid levels, Gauss-Newton iterations per level (finest first), correspondence gates,
    the lost-frame threshold, convergence thresholds and the model source."""
    _fields_ = [("levels", C.c_int32), ("iterations", C.c_int32 * 4), ("max_point_distance", C.c_float),
                ("max_normal_angle_deg", C.c_float), ("min_inlier_fraction", C.c_float),
                ("convergence_rotation", C.c_float), ("convergence_translation", C.c_float),
                ("model_source", C.c_int32)]

    @classmethod
    def defaults(cls) -> "TrackParams":
        return cls(3, (C.c_int32 * 4)(4, 5, 10, 0), 0.05, 20.0, 0.1, 1e-5, 1e-5, TRACK_CLOUD)


class TrackResult(C.Structure):
    """sm_track_result: tracked (0 = lost), steps applied, and the level-0 inliers, valid pixels and RMS residual."""
    _fields_ = [("tracked", C.c_int32), ("iterations", C.c_int32), ("inliers", C.c_uint32),
                ("valid_pixels", C.c_uint32), ("rms_residual", C.c_float)]


class TrackRGBDParams(C.Structure):
    """sm_track_rgbd_params: the photometric weight lambda (metres per intensity unit; 0 = the depth-only system), the
    |r_c| gate (intensity units, 0..255 scale) and the |grad I| gate (intensity units per pixel)."""
    _fields_ = [("photometric_weight", C.c_float), ("max_intensity_residual", C.c_float), ("min_gradient", C.c_float)]

    @classmethod
    def defaults(cls) -> "TrackRGBDParams":
        return cls(1e-4, 40.0, 2.0)


class TrackRGBDResult(C.Structure):
    """sm_track_rgbd_result: the depth-only TrackResult, and the level-0 photometric inliers and RMS intensity
    residual."""
    _fields_ = [("depth", TrackResult), ("photometric_inliers", C.c_uint32), ("rms_intensity", C.c_float)]


class MeshParams(C.Structure):
    """sm_mesh_params: k-NN radius factor, normal gate and largest triangle angle (main.cc's meshing defaults)."""
    _fields_ = [("neighbor_radius_factor", C.c_float), ("max_angle_between_normals_deg", C.c_float),
                ("max_triangle_angle_deg", C.c_float)]

    @classmethod
    def defaults(cls) -> "MeshParams":
        return cls(2.0, 90.0, 170.0)


class MeshStats(C.Structure):
    """sm_mesh_stats: triangles (also when the capacity was too small), meshed slots, boundary edges, overflows."""
    _fields_ = [("triangle_count", C.c_uint64), ("vertices_meshed", C.c_uint64), ("boundary_edges", C.c_uint64),
                ("umbrella_overflows", C.c_uint64)]


class MeshUpdateStats(C.Structure):
    """sm_mesh_update_stats: the whole mesh after the update, |C|, |A|, |R|, the delta sizes, and whether the
    umbrellas were rebuilt by the plain sweep."""
    _fields_ = [("mesh", MeshStats), ("slots_changed", C.c_uint64), ("umbrellas_rebuilt", C.c_uint64),
                ("owners_rechecked", C.c_uint64), ("triangles_added", C.c_uint64),
                ("triangles_removed", C.c_uint64), ("full_sweep", C.c_int32), ("reserved", C.c_int32)]


RELOC_MAX_CANDIDATES = 8


class RelocParams(C.Structure):
    """sm_reloc_params: the fern image level, fern count, table seed and depth-threshold range (metres), the keyframe
    capacity, the add and query bounds (fractions of the fern count), the candidates tried, the tracking parameters
    of a relocalisation attempt and its acceptance thresholds (inlier fraction, RMS residual in metres)."""
    _fields_ = [("level", C.c_int32), ("ferns", C.c_int32), ("seed", C.c_uint64), ("min_depth", C.c_float),
                ("max_depth", C.c_float), ("capacity", C.c_uint32), ("add_fraction", C.c_float),
                ("candidates", C.c_int32), ("max_query_fraction", C.c_float), ("track", TrackParams),
                ("accept_inlier_fraction", C.c_float), ("accept_rms", C.c_float)]

    @classmethod
    def defaults(cls) -> "RelocParams":
        track = TrackParams.defaults()
        track.max_point_distance = 0.1
        return cls(3, 512, 20150401, 0.3, 4.0, 4096, 0.2, 1, 0.4, track, 0.7, 0.01)


class RelocResult(C.Structure):
    """sm_reloc_result: relocalised (0 = the pose is NaN), tracking attempts, the accepted keyframe, its rank and
    distance (-1 / -1 / 0 when none), and the accepted attempt's TrackResult (the last attempt's otherwise)."""
    _fields_ = [("relocalised", C.c_int32), ("attempts", C.c_int32), ("keyframe", C.c_int32), ("rank", C.c_int32),
                ("distance", C.c_uint32), ("track", TrackResult)]


MESH_MAX_UMBRELLA = 16
MESH_ALL, MESH_ADDED, MESH_REMOVED = 0, 1, 2
MESH_MAX_HOLE = 16


class HoleParams(C.Structure):
    """sm_hole_params: the longest boundary loop filled (edges), the normal gate and the largest triangle angle."""
    _fields_ = [("max_hole_edges", C.c_int32), ("max_angle_between_normals_deg", C.c_float),
                ("max_triangle_angle_deg", C.c_float)]

    @classmethod
    def defaults(cls) -> "HoleParams":
        return cls(8, 90.0, 180.0)


class HoleStats(C.Structure):
    """sm_hole_stats: boundary edges of the input, loops found / filled / rejected / conflicting, triangles added
    (also when the capacity was too small) and the boundary edges of input and fill together."""
    _fields_ = [("boundary_edges", C.c_uint64), ("loops_found", C.c_uint64), ("loops_filled", C.c_uint64),
                ("loops_rejected", C.c_uint64), ("loops_conflicting", C.c_uint64), ("triangles_added", C.c_uint64),
                ("boundary_edges_after", C.c_uint64)]


MESH_MAX_VALENCE = 32
SIMPLIFY_MAX_ROUNDS = 1024
SIMPLIFY_STOP_TARGET, SIMPLIFY_STOP_CONVERGED, SIMPLIFY_STOP_MAX_ROUNDS = 1, 2, 3


class SimplifyParams(C.Structure):
    """sm_simplify_params: the triangle budget (0: none), the largest collapse cost (m^2), the normal gate, the
    largest triangle angle and the most rounds."""
    _fields_ = [("target_triangles", C.c_uint64), ("max_cost", C.c_double),
                ("max_angle_between_normals_deg", C.c_float), ("max_triangle_angle_deg", C.c_float),
                ("max_rounds", C.c_int32), ("reserved", C.c_int32)]

    @classmethod
    def defaults(cls, **overrides) -> "SimplifyParams":
        p = cls(0, 1e-6, 90.0, 170.0, 64, 0)
        for k, v in overrides.items():
            setattr(p, k, v)
        return p


class SimplifyStats(C.Structure):
    """sm_simplify_stats: triangles and corner slots in and out, collapses and rounds applied, the boundary edges
    (unchanged), the largest cost applied (m^2) and why the call stopped (SIMPLIFY_STOP_*)."""
    _fields_ = [("triangles_in", C.c_uint64), ("triangles_out", C.c_uint64), ("vertices_in", C.c_uint64),
                ("vertices_out", C.c_uint64), ("collapses", C.c_uint64), ("rounds", C.c_uint64),
                ("boundary_edges", C.c_uint64), ("max_cost_applied", C.c_double), ("stop_reason", C.c_int32),
                ("reserved", C.c_int32)]


TEXTURE_MAX_TILE = 512
TEXTURE_MAX_VIEWS = 1024
TEXTURE_MAX_ATLAS_SIDE = 32768


class TextureParams(C.Structure):
    """sm_texture_params: metres per texel, the largest atlas side, the most oblique view that contributes (degrees)
    and the relative depth tolerance of the visibility test."""
    _fields_ = [("texel_size", C.c_float), ("max_atlas_side", C.c_int32), ("max_view_angle_deg", C.c_float),
                ("depth_tolerance", C.c_float)]

    @classmethod
    def defaults(cls, **overrides) -> "TextureParams":
        p = cls(0.004, 16384, 75.0, 0.01)
        for k, v in overrides.items():
            setattr(p, k, v)
        return p


class TextureStats(C.Structure):
    """sm_texture_stats: triangles, the atlas size, the texels of all half-tiles, those some view saw and those that
    took the corner blend, the tiles capped at TEXTURE_MAX_TILE and the views that contributed."""
    _fields_ = [("triangles", C.c_uint64), ("atlas_width", C.c_int32), ("atlas_height", C.c_int32),
                ("texels", C.c_uint64), ("texels_seen", C.c_uint64), ("texels_fallback", C.c_uint64),
                ("tiles_clamped", C.c_uint64), ("views_used", C.c_uint64)]


class TextureViewDesc(C.Structure):
    """sm_texture_view: the camera (as sm_render_mesh takes it), view_T_global (3x4 row-major) and the device colour
    image (packed u8x3 rows) with its pitch in bytes."""
    _fields_ = [("camera", RenderParams), ("view_T_global", C.c_float * 12), ("color", C.c_void_p),
                ("color_pitch", C.c_size_t)]


class TextureGainParams(C.Structure):
    """sm_texture_gain_params: the most samples (points x views) of the gain fit, the conjugate-gradient steps
    (0: every gain 1), the noise and gain sigmas of the objective, and the levels outside which a sample takes no
    part in the fit."""
    _fields_ = [("max_samples", C.c_int32), ("iterations", C.c_int32), ("sigma_noise", C.c_float),
                ("sigma_gain", C.c_float), ("min_level", C.c_float), ("max_level", C.c_float)]

    @classmethod
    def defaults(cls, **overrides) -> "TextureGainParams":
        p = cls(1 << 23, 32, 10.0, 1.0, 5.0, 250.0)
        for k, v in overrides.items():
            setattr(p, k, v)
        return p


class TextureGainStats(C.Structure):
    """sm_texture_gain_stats: the sample points, the (point, view) samples in the fit, the views fitted, and the rms
    residual in grey levels at gain 1 and at the fitted gains."""
    _fields_ = [("points", C.c_uint64), ("samples", C.c_uint64), ("views_fitted", C.c_uint64),
                ("rms_before", C.c_double), ("rms_after", C.c_double)]


class ComponentParams(C.Structure):
    """sm_component_params: the fewest triangles and the least area (m^2) of a kept piece, and how many of the
    largest pieces may be kept (0: no limit)."""
    _fields_ = [("min_triangles", C.c_uint64), ("min_area", C.c_double), ("keep_largest", C.c_uint64)]

    @classmethod
    def defaults(cls, **overrides) -> "ComponentParams":
        p = cls(10, 0.0, 0)
        for k, v in overrides.items():
            setattr(p, k, v)
        return p


class ComponentStats(C.Structure):
    """sm_component_stats: triangles in and out, pieces and pieces kept, and the triangle count and area (m^2) of the
    largest piece."""
    _fields_ = [("triangles_in", C.c_uint64), ("triangles_out", C.c_uint64), ("components", C.c_uint64),
                ("components_kept", C.c_uint64), ("largest_triangles", C.c_uint64), ("largest_area", C.c_double)]


class MeshComponent(C.Structure):
    """sm_mesh_component: one piece's triangle count, area (m^2), smooth-position bounds, smallest triangle position
    and whether it is kept."""
    _fields_ = [("triangles", C.c_uint64), ("area", C.c_double), ("lo", C.c_float * 3), ("hi", C.c_float * 3),
                ("first_triangle", C.c_uint32), ("kept", C.c_int32)]


class CompactStats(C.Structure):
    """sm_compact_stats: surfels_size() before and after, the merged slots removed, the neighbour links of kept slots
    that named a removed slot, and whether the persistent sm_mesh_update mesh was carried over."""
    _fields_ = [("slots_before", C.c_uint64), ("slots_after", C.c_uint64), ("merged_removed", C.c_uint64),
                ("links_dropped", C.c_uint64), ("mesh_remapped", C.c_int32), ("reserved", C.c_int32)]


_P = C.c_void_p
_SZ = C.c_size_t
_F = C.c_float
_I = C.c_int32
_U16 = C.c_uint16
_U32 = C.c_uint32

# name -> (restype, argtypes); names without the prefix.
_SIGNATURES = {
    "last_error": (C.c_char_p, []),
    "version": (C.c_char_p, []),
    "create": (C.c_int, [C.POINTER(_P), C.c_uint64, _I, _I, _F, _F, _F, _F]),
    "destroy": (C.c_int, [_P]),
    "reset": (C.c_int, [_P, _P]),
    "preprocess": (C.c_int, [_P, _P, C.POINTER(PreprocessParams), _P, _SZ, C.POINTER(_P), C.POINTER(_SZ), _P,
                             _P, _SZ, _P, _SZ, _P, _SZ]),
    "bilateral_filter_and_depth_cutoff": (C.c_int, [_P, _F, _F, _U16, _F, _U16, _F, _I, _I, _P, _SZ, _P, _SZ]),
    "outlier_depth_map_fusion": (C.c_int, [_P, _I, _I, _F, _F, _F, _F, _F, _I, _I, _P, _SZ, C.POINTER(_P),
                                           C.POINTER(_SZ), _P, _P, _SZ]),
    "erode_depth_map": (C.c_int, [_P, _I, _I, _I, _P, _SZ, _P, _SZ]),
    "compute_normals_and_drop_bad_pixels": (C.c_int, [_P, _F, _F, _F, _F, _F, _F, _I, _I, _P, _SZ, _P, _SZ, _P, _SZ]),
    "compute_point_radii_and_remove_isolated_pixels": (C.c_int, [_P, _F, _F, _F, _F, _F, _F, _F, _I, _I, _P, _SZ,
                                                                 _P, _SZ, _P, _SZ]),
    "integrate": (C.c_int, [_P, _P, _U32, C.POINTER(IntegrateParams), _P, _SZ, _P, _SZ, _P, _SZ, _P, _SZ, _P, _P]),
    "regularize": (C.c_int, [_P, _P, _U32, _F, _F, _I]),
    "surfel_count": (C.c_int, [_P, C.POINTER(_U32)]),
    "surfels_size": (C.c_int, [_P, C.POINTER(_U32)]),
    "transfer_all_to_cpu": (C.c_int, [_P, _P, _U32, _P, _P, _P, _P, _P, _P, _P, _P, C.POINTER(C.c_uint64)]),
    "export_vertices": (C.c_int, [_P, _P, _P, _P]),
    "update_visualization_buffers": (C.c_int, [_P, _P, C.POINTER(VisualizationParams), _P, _P, _P]),
    "get_timings": (C.c_int, [_P, C.POINTER(_F * 7)]),
    "enable_timings": (C.c_int, [_P, _I]),
    "dump_state": (C.c_int, [_P, _P, _P, C.c_uint64, C.POINTER(_U32), C.POINTER(_U32)]),
    "load_state": (C.c_int, [_P, _P, _P, C.c_uint64, _U32, _U32]),
    "download_rasters": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "stream_run": (C.c_int, [_P, _P, C.POINTER(StreamDesc), C.POINTER(PreprocessParams), C.POINTER(IntegrateParams),
                             _I, _I, C.POINTER(StreamStats)]),
}
# Only the product exports these.
_PRODUCT_ONLY = {
    "default_integrate_params": (None, [C.POINTER(IntegrateParams)]),
    "default_preprocess_params": (None, [C.POINTER(PreprocessParams)]),
    "kernel_launch_count": (C.c_uint64, []),
    "profile_kernels": (C.c_int, [_I]),
    "profile_kernel_count": (_I, []),
    "profile_kernel_name": (C.c_char_p, [_I]),
    "profile_report": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_uint64), _I]),
    "frame_counters": (C.c_int, [_P, _P, C.POINTER(C.c_uint64 * 4)]),
    "configure": (C.c_int, [_P, C.c_char_p, C.c_double]),
    "median_filter_and_densify_depth_map": (C.c_int, [_P, _I, _I, _I, _P, _SZ, _P, _SZ, _P, _SZ]),
    "downscale_using_median_while_excluding": (C.c_int, [_P, _U16, _I, _I, _P, _SZ, _I, _I, _P, _SZ]),
    "color_image_pyramid": (C.c_int, [_P, _I, _I, _I, _P, _SZ, _P, _SZ]),
    "transfer_delta_to_cpu": (C.c_int, [_P, _P, _U32, C.POINTER(TransferToken), _P, _P, _P, _P, _P, _P, _P, _P,
                                        C.POINTER(TransferStats)]),
    "knn_create": (C.c_int, [C.POINTER(_P), _U32]),
    "knn_destroy": (None, [_P]),
    "knn_build": (C.c_int, [_P, _P, _U32, _P, _P, _P, _P, _P, _F]),
    "knn_build_from_reconstruction": (C.c_int, [_P, _P, _P, _F, C.POINTER(_U32)]),
    "knn_query": (C.c_int, [_P, _P, _U32, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "knn_batch_host": (C.c_int, [_P, _P, _U32, _P, _P, _P, _P, _F, _F, _I, _P, _P, _P]),
    "timeline_enable": (C.c_int, [_P, _I]),
    "timeline_read": (C.c_int, [_P, C.POINTER(C.c_uint64), _I]),
    "outlier_filter_transforms": (C.c_int, [_I, _F, _I, _P, _P, _I, _P]),
    "session_begin": (C.c_int, [_P, _P, C.POINTER(PreprocessParams), C.POINTER(IntegrateParams), _I, _I, _U32]),
    "session_push": (C.c_int, [_P, _P, _SZ, _P, _SZ, _I, _P, _P, C.POINTER(SessionStatus)]),
    "session_end": (C.c_int, [_P, C.POINTER(StreamStats)]),
    "render_surfels": (C.c_int, [_P, _P, C.POINTER(RenderParams), _P, _P, _SZ, _P, _SZ, _P, _SZ, _P, _SZ]),
    "render_mesh": (C.c_int, [_P, _P, C.POINTER(RenderParams), _P, _P, C.c_uint64, _I, _P, _SZ, _P, _SZ, _P, _SZ, _P,
                              _SZ]),
    "render_mesh_textured": (C.c_int, [_P, _P, C.POINTER(RenderParams), _P, _P, C.c_uint64, _I, _P, _P, _SZ, _I, _I,
                                       _P, _SZ, _P, _SZ, _P, _SZ, _P, _SZ]),
    "default_track_params": (None, [C.POINTER(TrackParams)]),
    "track_frame": (C.c_int, [_P, _P, C.POINTER(TrackParams), C.POINTER(PreprocessParams), _P, _SZ, _P, _P,
                              C.POINTER(TrackResult)]),
    "track_linearize": (C.c_int, [_P, _P, C.POINTER(TrackParams), _I, _F, _P, _SZ, _P, _SZ, _P, _SZ, _P, _P,
                                  C.POINTER(_U32)]),
    "default_track_rgbd_params": (None, [C.POINTER(TrackRGBDParams)]),
    "track_frame_rgbd": (C.c_int, [_P, _P, C.POINTER(TrackParams), C.POINTER(PreprocessParams),
                                   C.POINTER(TrackRGBDParams), _P, _SZ, _P, _SZ, _P, _P, C.POINTER(TrackRGBDResult)]),
    "track_linearize_rgbd": (C.c_int, [_P, _P, C.POINTER(TrackParams), C.POINTER(TrackRGBDParams), _I, _F, _P, _SZ,
                                       _P, _SZ, _P, _SZ, _P, _SZ, _P, _SZ, _P, _P, C.POINTER(C.c_double),
                                       C.POINTER(_U32), C.POINTER(_U32)]),
    "default_mesh_params": (None, [C.POINTER(MeshParams)]),
    "triangulate": (C.c_int, [_P, _P, C.POINTER(MeshParams), _P, C.c_uint64, C.POINTER(MeshStats)]),
    "mesh_update": (C.c_int, [_P, _P, C.POINTER(MeshParams), C.POINTER(MeshUpdateStats)]),
    "mesh_read": (C.c_int, [_P, _P, _I, _P, C.c_uint64, C.POINTER(C.c_uint64)]),
    "default_hole_params": (None, [C.POINTER(HoleParams)]),
    "mesh_fill_holes": (C.c_int, [_P, _P, C.POINTER(HoleParams), _P, C.c_uint64, _P, C.c_uint64, C.POINTER(HoleStats)]),
    "default_reloc_params": (None, [C.POINTER(RelocParams)]),
    "keyframe_db_create": (C.c_int, [C.POINTER(_P), _P, C.POINTER(RelocParams)]),
    "keyframe_db_destroy": (None, [_P]),
    "keyframe_db_reset": (C.c_int, [_P]),
    "keyframe_db_count": (C.c_int, [_P, C.POINTER(_U32)]),
    "keyframe_db_encode": (C.c_int, [_P, _P, _P, _SZ, _P, _SZ, _F, _P]),
    "keyframe_db_add": (C.c_int, [_P, _P, _P, _SZ, _P, _SZ, _F, _P, _I, C.POINTER(_I), C.POINTER(_I)]),
    "keyframe_db_query": (C.c_int, [_P, _P, _P, _SZ, _P, _SZ, _F, _P, _P, C.POINTER(_I)]),
    "keyframe_db_read": (C.c_int, [_P, _U32, _P, _P]),
    "relocalise": (C.c_int, [_P, _P, _P, C.POINTER(RelocParams), C.POINTER(PreprocessParams),
                             C.POINTER(TrackRGBDParams), _P, _SZ, _P, _SZ, _P, C.POINTER(RelocResult)]),
    "compact": (C.c_int, [_P, _P, _P, C.c_uint64, C.POINTER(CompactStats)]),
    "default_simplify_params": (None, [C.POINTER(SimplifyParams)]),
    "mesh_simplify": (C.c_int, [_P, _P, C.POINTER(SimplifyParams), _P, C.c_uint64, _P, C.c_uint64,
                                C.POINTER(SimplifyStats)]),
    "default_texture_params": (None, [C.POINTER(TextureParams)]),
    "mesh_texture": (C.c_int, [_P, _P, C.POINTER(TextureParams), _P, C.c_uint64, C.POINTER(TextureViewDesc), _I, _P,
                               _SZ, _I, _I, _P, C.POINTER(TextureStats)]),
    "default_texture_gain_params": (None, [C.POINTER(TextureGainParams)]),
    "mesh_texture_compensated": (C.c_int, [_P, _P, C.POINTER(TextureParams), C.POINTER(TextureGainParams), _P,
                                           C.c_uint64, C.POINTER(TextureViewDesc), _I, _P, _SZ, _I, _I, _P, _P,
                                           C.POINTER(TextureStats), C.POINTER(TextureGainStats)]),
    "default_component_params": (None, [C.POINTER(ComponentParams)]),
    "mesh_components": (C.c_int, [_P, _P, C.POINTER(ComponentParams), _P, C.c_uint64, _P, C.c_uint64, _P, _P,
                                  C.c_uint64, C.POINTER(ComponentStats)]),
}

EXPORTED_SYMBOLS = sorted(["sm_" + n for n in list(_SIGNATURES) + list(_PRODUCT_ONLY)])


class SurfelError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"[{code}] {message}")
        self.code = code


class Library:
    """One loaded shared library exporting the surfel C ABI under `prefix`."""

    def __init__(self, path: Path, prefix: str, product: bool):
        if not Path(path).exists():
            raise ImportError(
                f"{path} is missing. Build it with `python -m surfelmeshing_b200.build` "
                "(or __graft_entry__.build()); there is no CPU fallback for the surfel kernels.")
        self.path = Path(path)
        self.prefix = prefix
        self.cdll = C.CDLL(str(path), mode=C.RTLD_LOCAL)
        self.fn = {}
        sigs = dict(_SIGNATURES)
        if product:
            sigs.update(_PRODUCT_ONLY)
        for name, (restype, argtypes) in sigs.items():
            f = getattr(self.cdll, prefix + name)  # AttributeError if the symbol is not exported
            f.restype = restype
            f.argtypes = argtypes
            self.fn[name] = f

    def call(self, name: str, *args):
        """Calls a status-returning entry point and raises SurfelError on failure."""
        status = self.fn[name](*args)
        if status != SM_OK:
            raise self.error(status)
        return status

    def error(self, status: int) -> SurfelError:
        """The SurfelError of a failed status an entry point returned, with the library's last error message."""
        return SurfelError(status, self.fn["last_error"]().decode(errors="replace"))

    def version(self) -> str:
        return self.fn["version"]().decode()


_product: Library | None = None
_reference: Library | None = None
_shimref: Library | None = None


def load_product() -> Library:
    """The product library. SM_B200_LIB=<path> loads another BUILD OF THE PRODUCT instead (A/B
    measurements of kernel variants, e.g. variants/lib_x.so from
    `python -m surfelmeshing_b200.build --out variants/lib_x.so -- <nvcc flags>`); it exports the same ABI."""
    global _product
    if _product is None:
        import os
        override = os.environ.get("SM_B200_LIB")
        _product = Library(Path(override).resolve() if override else LIB_PATH, "sm_", product=True)
    return _product


def load_reference_oracle() -> Library:
    """TEST INFRASTRUCTURE ONLY: the reference's kernels behind the same ABI."""
    global _reference
    if _reference is None:
        _reference = Library(REF_LIB_PATH, "smref_", product=False)
    return _reference


def load_shim_oracle() -> Library:
    """TEST INFRASTRUCTURE ONLY: reference host glue + vis:: link shims -> the product's kernels."""
    global _shimref
    if _shimref is None:
        load_product()  # the shim library links against libsurfel_b200.so
        C.CDLL(str(LIB_PATH), mode=C.RTLD_GLOBAL)
        _shimref = Library(SHIM_LIB_PATH, "smref_", product=False)
    return _shimref
