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


MESH_MAX_UMBRELLA = 16

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
    "default_track_params": (None, [C.POINTER(TrackParams)]),
    "track_frame": (C.c_int, [_P, _P, C.POINTER(TrackParams), C.POINTER(PreprocessParams), _P, _SZ, _P, _P,
                              C.POINTER(TrackResult)]),
    "track_linearize": (C.c_int, [_P, _P, C.POINTER(TrackParams), _I, _F, _P, _SZ, _P, _SZ, _P, _SZ, _P, _P,
                                  C.POINTER(_U32)]),
    "default_mesh_params": (None, [C.POINTER(MeshParams)]),
    "triangulate": (C.c_int, [_P, _P, C.POINTER(MeshParams), _P, C.c_uint64, C.POINTER(MeshStats)]),
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
            raise SurfelError(status, self.fn["last_error"]().decode(errors="replace"))
        return status

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
