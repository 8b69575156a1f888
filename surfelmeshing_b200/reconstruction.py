"""Host-side mirror of the reference interface for the surfel reconstruction hot path.

`CUDASurfelReconstruction` has the public surface of the reference class of the same
name (applications/surfel_meshing/src/surfel_meshing/cuda_surfel_reconstruction.h:44-176):
Integrate / Regularize / TransferAllToCPU / ExportVertices / GetTimings / surfel_count /
surfels_size, same argument order and meaning. The depth pre-processing free functions
keep the reference's names (cuda_depth_processing.cuh:43-122). Everything forwards to the
C ABI (include/surfel_b200.h); PyTorch only provides device memory and streams.

The same class drives the parity oracle when constructed with
`lib=load_reference_oracle()` (tests / bench reference arm only).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from . import mesh_io
from ._lib import (CompactStats, ComponentParams, ComponentStats, HoleParams, HoleStats, IntegrateParams, SimplifyParams, SimplifyStats, Library, MeshComponent, MeshParams, MeshStats, MeshUpdateStats,
                   PreprocessParams, RelocParams, RelocResult, RenderParams, SessionStatus, StreamDesc, StreamStats,
                   TextureParams, TextureStats, TextureViewDesc, TrackParams, TrackResult,
                   TrackRGBDParams, TrackRGBDResult,
                   TransferStats, TransferToken, VisualizationParams)

RENDER_OUTPUTS = ("depth", "color", "normal", "index")

BUFFER_NAMES = ["surfel_x_buffer", "surfel_y_buffer", "surfel_z_buffer", "surfel_radius_squared_buffer",
                "surfel_normal_x_buffer", "surfel_normal_y_buffer", "surfel_normal_z_buffer",
                "surfel_last_update_stamp_buffer"]


def make_cpu_buffers(max_surfel_count: int, pinned: bool = False) -> dict:
    """The eight arrays of CUDASurfelBuffersCPU (APP/cuda_surfels_cpu.h:40-73), max_surfel_count long."""
    out = {}
    for k in BUFFER_NAMES:
        dtype = np.uint32 if "stamp" in k else np.float32
        if pinned:
            t = torch.empty(max(max_surfel_count, 1), dtype=torch.int32 if "stamp" in k else torch.float32).pin_memory()
            out[k] = t.numpy().view(dtype)
            out["_keep_" + k] = t
        else:
            out[k] = np.zeros(max(max_surfel_count, 1), dtype=dtype)
    return out

ROW_NAMES = [
    "x", "y", "z", "smooth_x", "smooth_y", "smooth_z", "confidence", "radius_squared",
    "normal_x", "normal_y", "normal_z", "gradient_x", "gradient_y", "gradient_z",
    "accum_x", "accum_y", "accum_z", "creation_stamp", "last_update_stamp",
    "neighbor0", "neighbor1", "neighbor2", "neighbor3", "gradient_count", "color",
]
# Rows that hold scratch data between calls and are excluded from state comparisons:
# gradient (11-13), accum (14-16, never written), gradient weight sum (23).
SCRATCH_ROWS = (11, 12, 13, 14, 15, 16, 23)


def _stream_handle(stream) -> int:
    if stream is None:
        return torch.cuda.current_stream().cuda_stream
    if isinstance(stream, torch.cuda.Stream):
        return stream.cuda_stream
    return int(stream)


def _raster(t: torch.Tensor, channels: int = 1):
    """(device pointer, pitch in bytes) of a row-pitched raster tensor [H, W(, C)]."""
    if not t.is_cuda:
        raise ValueError("rasters must be CUDA tensors (there is no CPU path)")
    if channels == 1:
        assert t.dim() == 2 and t.stride(1) == 1, "expected [H, W] raster with unit pixel stride"
    else:
        assert t.dim() == 3 and t.shape[2] == channels and t.stride(2) == 1 and t.stride(1) == channels
    return C.c_void_p(t.data_ptr()), t.stride(0) * t.element_size()


def _check_triangles(triangles) -> None:
    """The triangle list of the mesh calls: an int32 CUDA tensor [T, 3] of slot indices."""
    if not (isinstance(triangles, torch.Tensor) and triangles.is_cuda and triangles.dtype == torch.int32
            and triangles.dim() == 2 and triangles.shape[1] == 3):
        raise ValueError("triangles must be an int32 CUDA tensor [T, 3]")


def _check_texture(texture, count: int):
    """The (atlas, uv) pair of a textured render_mesh(): atlas uint8 CUDA [H, W, 3] with packed rows, uv float32 CUDA
    [T, 3, 2] for a list of `count` triangles. Returns (atlas, contiguous uv)."""
    if not (isinstance(texture, (tuple, list)) and len(texture) == 2):
        raise ValueError("texture must be the (atlas, uv) pair that texture_mesh() returns")
    atlas, uv = texture
    if not (isinstance(atlas, torch.Tensor) and atlas.is_cuda and atlas.dtype == torch.uint8 and atlas.dim() == 3
            and atlas.shape[2] == 3 and atlas.stride(2) == 1 and atlas.stride(1) == 3):
        raise ValueError("the atlas must be a uint8 CUDA tensor [H, W, 3] with packed rows")
    if not (isinstance(uv, torch.Tensor) and uv.is_cuda and uv.dtype == torch.float32 and uv.dim() == 3
            and tuple(uv.shape[1:]) == (3, 2)):
        raise ValueError("uv must be a float32 CUDA tensor [T, 3, 2]")
    if uv.shape[0] != count:
        raise ValueError(f"uv has {uv.shape[0]} triangles, the list {count}")
    return atlas, uv.contiguous()


def _mat12(m) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(m, dtype=np.float32).reshape(-1)[:12])
    assert a.size == 12
    return a


def invert_rigid(m) -> np.ndarray:
    """Inverse of a 3x4 rigid transform, computed in float64 and rounded to float32 once."""
    a = np.asarray(m, dtype=np.float64).reshape(3, 4)
    R, t = a[:, :3], a[:, 3]
    return np.concatenate([R.T, (-R.T @ t)[:, None]], axis=1).astype(np.float32)


def shade_normals(normal: torch.Tensor) -> torch.Tensor:
    """The reference viewer's triangle-normal shading (--triangle_normal_shading, light = the viewing direction) of a
    camera-frame normal image [H, W, 3] from render_mesh(): intensity = clamp(0.8 * (-n.z) + 0.2, 0, 1) as uint8
    [H, W] (x 255, rounded); pixels whose normal is zero (empty) are 0."""
    if normal.dim() != 3 or normal.shape[2] != 3:
        raise ValueError("normal must be [H, W, 3]")
    n = normal.float()
    intensity = (0.8 * (-n[..., 2]) + 0.2).clamp(0.0, 1.0)
    value = torch.round(intensity * 255.0).to(torch.uint8)
    return torch.where((n != 0).any(dim=2), value, torch.zeros_like(value))


class TextureView:
    """One posed colour image for CUDASurfelReconstruction.texture_mesh(): a uint8 CUDA tensor [H, W, 3] (r, g, b,
    row-pitched), the synthetic.Camera it was taken with (pixel-corner intrinsics, size H x W), and its pose as
    view_T_global (global -> camera) or global_T_view (camera -> global; inverted in float64). Only surfaces with
    near <= camera depth <= far take colour from it."""

    def __init__(self, color: torch.Tensor, camera, view_T_global=None, global_T_view=None, near: float = 0.1,
                 far: float = 100.0):
        if (view_T_global is None) == (global_T_view is None):
            raise ValueError("give exactly one of view_T_global and global_T_view")
        if not (isinstance(color, torch.Tensor) and color.is_cuda and color.dtype == torch.uint8
                and tuple(color.shape) == (camera.height, camera.width, 3)):
            raise ValueError(f"color must be a uint8 CUDA tensor of shape {(camera.height, camera.width, 3)}")
        self.color = color if color.stride(2) == 1 and color.stride(1) == 3 else color.contiguous()
        self.camera = camera
        self.view_T_global = _mat12(view_T_global if view_T_global is not None else invert_rigid(global_T_view))
        self.near, self.far = float(near), float(far)

    def desc(self) -> TextureViewDesc:
        c = self.camera
        d = TextureViewDesc()
        d.camera = RenderParams(c.width, c.height, float(c.fx), float(c.fy), float(c.cx), float(c.cy), self.near,
                                self.far)
        d.view_T_global = (C.c_float * 12)(*self.view_T_global.tolist())
        d.color = self.color.data_ptr()
        d.color_pitch = self.color.stride(0)
        return d


# ---------------------------------------------------------------------------------------
# depth pre-processing (names of cuda_depth_processing.cuh)
# ---------------------------------------------------------------------------------------

def BilateralFilteringAndDepthCutoffCUDA(stream, sigma_xy, sigma_value_factor, value_to_ignore, radius_factor,
                                         max_depth, depth_valid_region_radius, input_depth, output_depth,
                                         lib: Optional[Library] = None):
    lib = lib or _lib.load_product()
    ip, ipitch = _raster(input_depth)
    op, opitch = _raster(output_depth)
    H, W = input_depth.shape
    lib.call("bilateral_filter_and_depth_cutoff", _stream_handle(stream), sigma_xy, sigma_value_factor,
             int(value_to_ignore), radius_factor, int(max_depth), depth_valid_region_radius, W, H, ip, ipitch,
             op, opitch)


def _others_args(other_depths: Sequence[torch.Tensor], others_TR_reference):
    K = len(other_depths)
    ptrs = (C.c_void_p * K)(*[t.data_ptr() for t in other_depths])
    pitches = (C.c_size_t * K)(*[t.stride(0) * t.element_size() for t in other_depths])
    mats = np.ascontiguousarray(np.asarray(others_TR_reference, dtype=np.float32).reshape(K, 12))
    return K, ptrs, pitches, mats


def OutlierDepthMapFusionCUDA(stream, tolerance, input_depth, depth_fx, depth_fy, depth_cx, depth_cy, other_depths,
                              others_TR_reference, output_depth, required_count: int = -1,
                              lib: Optional[Library] = None):
    """Both reference overloads: required_count = -1 means 'all other frames must agree'."""
    lib = lib or _lib.load_product()
    K, ptrs, pitches, mats = _others_args(other_depths, others_TR_reference)
    ip, ipitch = _raster(input_depth)
    op, opitch = _raster(output_depth)
    H, W = input_depth.shape
    lib.call("outlier_depth_map_fusion", _stream_handle(stream), K, required_count, tolerance, depth_fx, depth_fy,
             depth_cx, depth_cy, W, H, ip, ipitch, ptrs, pitches, mats.ctypes.data_as(C.c_void_p), op, opitch)


def MedianFilterAndDensifyDepthMap(stream, iterations, input_depth, output_depth=None, lib: Optional[Library] = None):
    """APP/main.cc:207-252 (there on the CPU, main.cc:927-939): `iterations` passes of the 3x3
    zero-excluding median that also fills holes. Returns the output tensor."""
    lib = lib or _lib.load_product()
    H, W = input_depth.shape
    if output_depth is None:
        output_depth = torch.zeros((H, W), dtype=torch.uint16, device=input_depth.device)
    scratch = torch.zeros((H, W), dtype=torch.uint16, device=input_depth.device)
    ip, ipitch = _raster(input_depth)
    op, opitch = _raster(output_depth)
    sp, spitch = _raster(scratch)
    lib.call("median_filter_and_densify_depth_map", _stream_handle(stream), int(iterations), W, H, ip, ipitch, op, opitch,
             sp, spitch)
    return output_depth


def DownscaleUsingMedianWhileExcluding(stream, value_to_ignore, output_width, output_height, input_depth,
                                       output_depth=None, lib: Optional[Library] = None):
    """Image<u16>::DownscaleUsingMedianWhileExcluding (libvis image.h:1003-1050; APP/main.cc:951-952, there on
    the CPU): each output pixel is the median of its input block without `value_to_ignore`. Returns the
    [output_height, output_width] output tensor."""
    lib = lib or _lib.load_product()
    H, W = input_depth.shape
    if output_depth is None:
        output_depth = torch.zeros((int(output_height), int(output_width)), dtype=torch.uint16,
                                   device=input_depth.device)
    ip, ipitch = _raster(input_depth)
    op, opitch = _raster(output_depth)
    lib.call("downscale_using_median_while_excluding", _stream_handle(stream), int(value_to_ignore), W, H, ip, ipitch,
             int(output_width), int(output_height), op, opitch)
    return output_depth


def ImagePyramid(stream, color, pyramid_level, output=None, lib: Optional[Library] = None):
    """ImagePyramid(color, pyramid_level) (libvis image_cache.h:205-282; APP/main.cc:973-981, there on the CPU):
    `pyramid_level` rounds of DownscaleToHalfSize on a [H, W, 3] uint8 image. Returns the
    [H >> level, W >> level, 3] output tensor."""
    lib = lib or _lib.load_product()
    H, W = color.shape[:2]
    level = int(pyramid_level)
    if output is None:
        output = torch.zeros((max(H >> level, 1), max(W >> level, 1), 3), dtype=torch.uint8, device=color.device)
    ip, ipitch = _raster(color, 3)
    op, opitch = _raster(output, 3)
    lib.call("color_image_pyramid", _stream_handle(stream), level, W, H, ip, ipitch, op, opitch)
    return output


def ErodeDepthMapCUDA(stream, radius, input_depth, output_depth, lib: Optional[Library] = None):
    lib = lib or _lib.load_product()
    ip, ipitch = _raster(input_depth)
    op, opitch = _raster(output_depth)
    H, W = input_depth.shape
    lib.call("erode_depth_map", _stream_handle(stream), radius, W, H, ip, ipitch, op, opitch)


def CopyWithoutBorderCUDA(stream, input_depth, output_depth, lib: Optional[Library] = None):
    ErodeDepthMapCUDA(stream, 0, input_depth, output_depth, lib=lib)


def ComputeNormalsAndDropBadPixelsCUDA(stream, observation_angle_threshold_deg, depth_scaling, depth_fx, depth_fy,
                                       depth_cx, depth_cy, in_depth, out_depth, out_normals,
                                       lib: Optional[Library] = None):
    lib = lib or _lib.load_product()
    ip, ipitch = _raster(in_depth)
    op, opitch = _raster(out_depth)
    np_, npitch = _raster(out_normals, 2)
    H, W = in_depth.shape
    lib.call("compute_normals_and_drop_bad_pixels", _stream_handle(stream), observation_angle_threshold_deg,
             depth_scaling, depth_fx, depth_fy, depth_cx, depth_cy, W, H, ip, ipitch, op, opitch, np_, npitch)


def ComputePointRadiiAndRemoveIsolatedPixelsCUDA(stream, point_radius_extension_factor, point_radius_clamp_factor,
                                                 depth_scaling, depth_fx, depth_fy, depth_cx, depth_cy, depth_buffer,
                                                 radius_buffer, out_depth, lib: Optional[Library] = None):
    lib = lib or _lib.load_product()
    ip, ipitch = _raster(depth_buffer)
    rp, rpitch = _raster(radius_buffer)
    op, opitch = _raster(out_depth)
    H, W = depth_buffer.shape
    lib.call("compute_point_radii_and_remove_isolated_pixels", _stream_handle(stream),
             point_radius_extension_factor, point_radius_clamp_factor, depth_scaling, depth_fx, depth_fy, depth_cx,
             depth_cy, W, H, ip, ipitch, rp, rpitch, op, opitch)


# ---------------------------------------------------------------------------------------
# CUDASurfelReconstruction
# ---------------------------------------------------------------------------------------

class CUDASurfelReconstruction:
    """Mirror of vis::CUDASurfelReconstruction (cuda_surfel_reconstruction.h:44-176).

    The constructor takes the camera as (width, height, fx, fy, cx, cy) with cx, cy in the
    reference's pixel-corner convention (PinholeCamera4f::parameters()); the three OpenGL
    resources and the render window of the reference constructor are GUI-only and omitted.
    """

    def __init__(self, max_surfel_count: int, width: int, height: int, fx: float, fy: float, cx: float, cy: float,
                 lib: Optional[Library] = None):
        self.lib = lib or _lib.load_product()
        self.width, self.height = int(width), int(height)
        self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
        self.max_surfel_count = int(max_surfel_count)
        handle = C.c_void_p()
        self.lib.call("create", C.byref(handle), self.max_surfel_count, self.width, self.height, self.fx, self.fy,
                      self.cx, self.cy)
        self._h = handle

    def close(self):
        if getattr(self, "_h", None):
            self.lib.fn["destroy"](self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- reference API ------------------------------------------------------------------
    def Integrate(self, stream, frame_index, depth_scaling, depth_buffer, normals_buffer, radius_buffer,
                  color_buffer, global_T_local, sensor_noise_factor, max_surfel_confidence, regularizer_weight,
                  regularization_frame_window_size, do_blending, measurement_blending_radius,
                  regularization_iterations_per_integration_iteration, radius_factor_for_regularization_neighbors,
                  normal_compatibility_threshold_deg, surfel_integration_active_window_size,
                  local_T_global=None):
        """cuda_surfel_reconstruction.cc:112-320. `depth_buffer` is blended in place.

        `local_T_global` defaults to the float64 inverse of `global_T_local` rounded to fp32
        (the reference inverts with Sophus on the host)."""
        p = IntegrateParams(depth_scaling, sensor_noise_factor, max_surfel_confidence, regularizer_weight,
                            regularization_frame_window_size, 1 if do_blending else 0, measurement_blending_radius,
                            regularization_iterations_per_integration_iteration,
                            radius_factor_for_regularization_neighbors, normal_compatibility_threshold_deg,
                            surfel_integration_active_window_size)
        self.integrate(stream, frame_index, p, depth_buffer, normals_buffer, radius_buffer, color_buffer,
                       global_T_local, local_T_global)

    def integrate(self, stream, frame_index, params: IntegrateParams, depth_buffer, normals_buffer, radius_buffer,
                  color_buffer, global_T_local, local_T_global=None):
        g = _mat12(global_T_local)
        l = _mat12(local_T_global if local_T_global is not None else invert_rigid(g))
        dp, dpitch = _raster(depth_buffer)
        np_, npitch = _raster(normals_buffer, 2)
        rp, rpitch = _raster(radius_buffer)
        cp, cpitch = _raster(color_buffer, 3)
        self.lib.call("integrate", self._h, _stream_handle(stream), int(frame_index), C.byref(params), dp, dpitch,
                      np_, npitch, rp, rpitch, cp, cpitch, g.ctypes.data_as(C.c_void_p),
                      l.ctypes.data_as(C.c_void_p))

    def Regularize(self, stream, frame_index, regularizer_weight, radius_factor_for_regularization_neighbors,
                   regularization_frame_window_size):
        """cuda_surfel_reconstruction.cc:322-337."""
        self.lib.call("regularize", self._h, _stream_handle(stream), int(frame_index), regularizer_weight,
                      radius_factor_for_regularization_neighbors, regularization_frame_window_size)

    def TransferAllToCPU(self, stream, frame_index, buffers: Optional[dict] = None) -> dict:
        """cuda_surfel_reconstruction.cc:339-359: fills the CUDASurfelBuffersCPU arrays
        (cuda_surfels_cpu.h:40-73) and returns them (synchronises the stream)."""
        n = self.surfels_size()
        names = ["surfel_x_buffer", "surfel_y_buffer", "surfel_z_buffer", "surfel_radius_squared_buffer",
                 "surfel_normal_x_buffer", "surfel_normal_y_buffer", "surfel_normal_z_buffer",
                 "surfel_last_update_stamp_buffer"]
        if buffers is None:
            buffers = {k: np.empty(max(n, 1), dtype=np.uint32 if "stamp" in k else np.float32) for k in names}
        count = C.c_uint64()
        ptrs = [buffers[k].ctypes.data_as(C.c_void_p) for k in names]
        self.lib.call("transfer_all_to_cpu", self._h, _stream_handle(stream), int(frame_index), *ptrs,
                      C.byref(count))
        torch.cuda.synchronize()
        buffers["frame_index"] = int(frame_index)
        buffers["surfel_count"] = int(count.value)
        return buffers

    def TransferDeltaToCPU(self, stream, frame_index, buffers: dict, token: TransferToken) -> TransferStats:
        """sm_transfer_delta_to_cpu: brings `buffers` (filled by the transfer `token` stands for; a fresh
        TransferToken() = never) up to date; afterwards they equal a full TransferAllToCPU. The arrays
        must be at least surfels_size() long (the reference allocates max_surfel_count)."""
        stats = TransferStats()
        ptrs = [buffers[k].ctypes.data_as(C.c_void_p) for k in BUFFER_NAMES]
        self.lib.call("transfer_delta_to_cpu", self._h, _stream_handle(stream), int(frame_index), C.byref(token), *ptrs,
                      C.byref(stats))
        buffers["frame_index"] = int(frame_index)
        buffers["surfel_count"] = int(stats.surfel_count)
        return stats

    def UpdateVisualizationBuffers(self, stream, frame_index, latest_triangulated_frame_index, latest_mesh_surfel_count,
                                   surfel_integration_active_window_size, visualize_last_update_timestamp,
                                   visualize_creation_timestamp, visualize_radii, visualize_normals,
                                   vertex_buffer=None, neighbor_index_buffer=None, normal_vertex_buffer=None,
                                   point_size_in_floats: int = 4):
        """cuda_surfel_reconstruction.cc:361-403; the three OpenGL buffers of the reference are plain
        device tensors here (None = not wanted)."""
        p = VisualizationParams(int(frame_index), int(latest_triangulated_frame_index), int(latest_mesh_surfel_count),
                                int(surfel_integration_active_window_size), int(point_size_in_floats),
                                int(bool(visualize_last_update_timestamp)), int(bool(visualize_creation_timestamp)),
                                int(bool(visualize_radii)), int(bool(visualize_normals)))
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        self.lib.call("update_visualization_buffers", self._h, _stream_handle(stream), C.byref(p), ptr(vertex_buffer),
                      ptr(neighbor_index_buffer), ptr(normal_vertex_buffer))

    def render(self, view_T_global, width: int, height: int, fx: float, fy: float, cx: float, cy: float,
               near: float = 0.1, far: float = 100.0, stream=None, outputs=RENDER_OUTPUTS) -> dict:
        """sm_render_surfels: the current cloud drawn as oriented disks (smooth position, normal, radius, colour)
        into a pinhole camera of any size; the nearest disk wins a pixel, equal depths the lower slot.

        view_T_global: 3x4 global-to-camera transform; fx, fy, cx, cy in the pixel-corner convention of the
        handle's camera; surfels with camera-space z outside [near, far] are not drawn. Returns the requested
        CUDA tensors, enqueued on `stream` (not synchronised): "depth" float32 [H, W] metres (0 = empty),
        "color" uint8 [H, W, 3], "normal" float32 [H, W, 3] camera-frame normal (0 = empty), "index" int32
        [H, W] surfel slot (-1 = empty)."""
        outputs = tuple(outputs)
        unknown = [o for o in outputs if o not in RENDER_OUTPUTS]
        if unknown or not outputs:
            raise ValueError(f"outputs must be a non-empty subset of {RENDER_OUTPUTS}, got {outputs}")
        H, W = int(height), int(width)
        shapes = {"depth": ((H, W), torch.float32), "color": ((H, W, 3), torch.uint8),
                  "normal": ((H, W, 3), torch.float32), "index": ((H, W), torch.int32)}
        out = {k: torch.empty(shapes[k][0], dtype=shapes[k][1], device="cuda") for k in outputs}
        if isinstance(stream, torch.cuda.Stream):
            for t in out.values():
                t.record_stream(stream)   # allocated on the current stream, written on `stream`
        args = []
        for k in RENDER_OUTPUTS:
            t = out.get(k)
            args += [C.c_void_p(t.data_ptr()), t.stride(0) * t.element_size()] if t is not None else [None, 0]
        p = RenderParams(W, H, float(fx), float(fy), float(cx), float(cy), float(near), float(far))
        T = _mat12(view_T_global)
        self.lib.call("render_surfels", self._h, _stream_handle(stream), C.byref(p), T.ctypes.data_as(C.c_void_p),
                      *args)
        return out

    def render_mesh(self, triangles, view_T_global, width: int, height: int, fx: float, fy: float, cx: float,
                    cy: float, near: float = 0.1, far: float = 100.0, unmeshed_surfels: bool = True, stream=None,
                    outputs=RENDER_OUTPUTS, texture=None) -> dict:
        """sm_render_mesh: a triangle list over the current cloud (the int32 CUDA tensor [T, 3] of slot indices that
        triangulate() and mesh_triangles() return) drawn into a pinhole camera of any size, with perspective-correct
        depth and colour; unmeshed_surfels=True also draws the slots no triangle names as disks, as render() does.
        Triangles naming merged or out-of-range slots, or with a corner outside [near, far], are not drawn.

        texture: the (atlas, uv) pair texture_mesh() returns for `triangles` (atlas uint8 CUDA [H, W, 3] with packed
        rows, uv float32 CUDA [T, 3, 2]); the triangles are then coloured by bilinear lookups in the atlas at
        perspective-correct texture coordinates (sm_render_mesh_textured), and "color" must be among the outputs.

        Returns the dict of render(): "depth", "color", "normal" (the unit triangle normal facing the camera) and
        "index" (the triangle's row in `triangles`; a disk's slot with bit 31 set, so negative in int32; -1 = empty),
        enqueued on `stream` (not synchronised)."""
        outputs = tuple(outputs)
        unknown = [o for o in outputs if o not in RENDER_OUTPUTS]
        if unknown or not outputs:
            raise ValueError(f"outputs must be a non-empty subset of {RENDER_OUTPUTS}, got {outputs}")
        _check_triangles(triangles)
        triangles = triangles.contiguous()
        count = int(triangles.shape[0])
        if texture is not None:
            atlas, uv = _check_texture(texture, count)
            if "color" not in outputs:
                raise ValueError("a textured render needs 'color' among the outputs")
        H, W = int(height), int(width)
        shapes = {"depth": ((H, W), torch.float32), "color": ((H, W, 3), torch.uint8),
                  "normal": ((H, W, 3), torch.float32), "index": ((H, W), torch.int32)}
        out = {k: torch.empty(shapes[k][0], dtype=shapes[k][1], device="cuda") for k in outputs}
        if isinstance(stream, torch.cuda.Stream):
            used = (*out.values(), triangles) if texture is None else (*out.values(), triangles, atlas, uv)
            for t in used:
                t.record_stream(stream)   # allocated on the current stream, used on `stream`
        args = []
        for k in RENDER_OUTPUTS:
            t = out.get(k)
            args += [C.c_void_p(t.data_ptr()), t.stride(0) * t.element_size()] if t is not None else [None, 0]
        p = RenderParams(W, H, float(fx), float(fy), float(cx), float(cy), float(near), float(far))
        T = _mat12(view_T_global)
        head = (self._h, _stream_handle(stream), C.byref(p), T.ctypes.data_as(C.c_void_p),
                C.c_void_p(triangles.data_ptr()) if count else None, count,
                _lib.RENDER_UNMESHED_SURFELS if unmeshed_surfels else 0)
        if texture is None:
            self.lib.call("render_mesh", *head, *args)
        else:
            self.lib.call("render_mesh_textured", *head, C.c_void_p(uv.data_ptr()) if count else None,
                          C.c_void_p(atlas.data_ptr()) if atlas.numel() else None, atlas.stride(0),
                          int(atlas.shape[1]), int(atlas.shape[0]), *args)
        return out

    def track(self, depth, guess, params: Optional[TrackParams] = None, pp: Optional[PreprocessParams] = None,
              source: str = "cloud", stream=None):
        """sm_track_frame: the camera-to-world pose of a raw depth map ([H, W] uint16 CUDA tensor at the handle's
        camera size) by point-to-plane ICP, starting from `guess` (3x4 camera-to-world). source="cloud" tracks
        against the cloud rendered from the guess, source="previous" against the previous track() call's frame.
        Synchronous. Returns (pose [3, 4] float32, TrackResult); a lost frame returns the guess with tracked = 0."""
        if source not in ("cloud", "previous"):
            raise ValueError(f"source must be 'cloud' or 'previous', got {source!r}")
        tp = TrackParams.defaults() if params is None else TrackParams.from_buffer_copy(params)
        tp.model_source = _lib.TRACK_CLOUD if source == "cloud" else _lib.TRACK_PREVIOUS_FRAME
        pp = pp if pp is not None else PreprocessParams.defaults()
        dp, dpitch = _raster(depth)
        if tuple(depth.shape) != (self.height, self.width) or depth.dtype != torch.uint16:
            raise ValueError(f"depth must be uint16 [{self.height}, {self.width}]")
        g = _mat12(guess)
        out = np.zeros(12, np.float32)
        result = TrackResult()
        self.lib.call("track_frame", self._h, _stream_handle(stream), C.byref(tp), C.byref(pp), dp, dpitch,
                      g.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.byref(result))
        return out.reshape(3, 4), result

    def track_linearize(self, level: int, live_depth, model_depth, model_normal, model_T_live,
                        params: Optional[TrackParams] = None, depth_scaling: float = 5000.0, stream=None):
        """sm_track_linearize: one point-to-plane linearisation of a filtered live level image against caller model
        images (depth [H, W] float32, normal [H, W, 3] float32 at the handle's camera). Synchronous. Returns
        (system float64 [27]: the 21 upper-triangle J^T J sums then the 6 J^T r sums, inlier count)."""
        tp = TrackParams.defaults() if params is None else params
        level = int(level)
        if not 0 <= level <= 3:
            raise ValueError(f"level must be in [0, 3], got {level}")
        factor = float(np.float32(1.0) / np.float32(2.0 ** level))   # Camera.scaled(level) sizes
        live_shape = (int(factor * self.height + 0.5), int(factor * self.width + 0.5))
        H, W = self.height, self.width
        for name, t, shape, dtype in (("live_depth", live_depth, live_shape, torch.uint16),
                                      ("model_depth", model_depth, (H, W), torch.float32),
                                      ("model_normal", model_normal, (H, W, 3), torch.float32)):
            if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape or t.dtype != dtype:
                got = (tuple(t.shape), t.dtype) if isinstance(t, torch.Tensor) else type(t).__name__
                raise ValueError(f"{name} must be a {dtype} tensor of shape {shape}, got {got}")
        lp, lpitch = _raster(live_depth)
        mp, mpitch = _raster(model_depth)
        np_, npitch = _raster(model_normal, 3)
        T = _mat12(model_T_live)
        system = np.zeros(27, np.float64)
        inliers = C.c_uint32()
        self.lib.call("track_linearize", self._h, _stream_handle(stream), C.byref(tp), int(level), float(depth_scaling),
                      lp, lpitch, mp, mpitch, np_, npitch, T.ctypes.data_as(C.c_void_p),
                      system.ctypes.data_as(C.c_void_p), C.byref(inliers))
        return system, int(inliers.value)

    def _check_raster(self, name, t, shape, dtype):
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape or t.dtype != dtype:
            got = (tuple(t.shape), t.dtype) if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"{name} must be a {dtype} tensor of shape {shape}, got {got}")

    def track_rgbd(self, depth, color, guess, params: Optional[TrackParams] = None,
                   rgbd: Optional[TrackRGBDParams] = None, pp: Optional[PreprocessParams] = None, source: str = "cloud",
                   stream=None):
        """sm_track_frame_rgbd: track() with the registered colour image as well (colour [H, W, 3] uint8 CUDA tensor,
        r, g, b): joint point-to-plane and photometric Gauss-Newton, which also pins down the motions a single plane or
        a corridor leaves free wherever the surface has texture. source="previous" needs the previous tracking call
        on this handle to have been a track_rgbd() call. Synchronous. Returns (pose [3, 4] float32,
        TrackRGBDResult); a lost frame returns the guess with depth.tracked = 0."""
        if source not in ("cloud", "previous"):
            raise ValueError(f"source must be 'cloud' or 'previous', got {source!r}")
        tp = TrackParams.defaults() if params is None else TrackParams.from_buffer_copy(params)
        tp.model_source = _lib.TRACK_CLOUD if source == "cloud" else _lib.TRACK_PREVIOUS_FRAME
        rp = TrackRGBDParams.defaults() if rgbd is None else rgbd
        pp = pp if pp is not None else PreprocessParams.defaults()
        self._check_raster("depth", depth, (self.height, self.width), torch.uint16)
        self._check_raster("color", color, (self.height, self.width, 3), torch.uint8)
        dp, dpitch = _raster(depth)
        cp, cpitch = _raster(color, 3)
        g = _mat12(guess)
        out = np.zeros(12, np.float32)
        result = TrackRGBDResult()
        self.lib.call("track_frame_rgbd", self._h, _stream_handle(stream), C.byref(tp), C.byref(pp), C.byref(rp), dp,
                      dpitch, cp, cpitch, g.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
                      C.byref(result))
        return out.reshape(3, 4), result

    def track_linearize_rgbd(self, level: int, live_depth, live_color, model_depth, model_normal, model_color,
                             model_T_live, params: Optional[TrackParams] = None,
                             rgbd: Optional[TrackRGBDParams] = None, depth_scaling: float = 5000.0, stream=None):
        """sm_track_linearize_rgbd: one joint linearisation of a filtered live level image with the raw live colour
        (uint8 [H, W, 3] at the handle's camera) against caller model images (depth, normal, colour at the handle's
        camera). Synchronous. Returns (system float64 [27], sum r_c^2, depth inliers, photometric inliers)."""
        tp = TrackParams.defaults() if params is None else params
        rp = TrackRGBDParams.defaults() if rgbd is None else rgbd
        level = int(level)
        if not 0 <= level <= 3:
            raise ValueError(f"level must be in [0, 3], got {level}")
        factor = float(np.float32(1.0) / np.float32(2.0 ** level))   # Camera.scaled(level) sizes
        live_shape = (int(factor * self.height + 0.5), int(factor * self.width + 0.5))
        H, W = self.height, self.width
        for name, t, shape, dtype in (("live_depth", live_depth, live_shape, torch.uint16),
                                      ("live_color", live_color, (H, W, 3), torch.uint8),
                                      ("model_depth", model_depth, (H, W), torch.float32),
                                      ("model_normal", model_normal, (H, W, 3), torch.float32),
                                      ("model_color", model_color, (H, W, 3), torch.uint8)):
            self._check_raster(name, t, shape, dtype)
        lp, lpitch = _raster(live_depth)
        lc, lcpitch = _raster(live_color, 3)
        mp, mpitch = _raster(model_depth)
        np_, npitch = _raster(model_normal, 3)
        mc, mcpitch = _raster(model_color, 3)
        T = _mat12(model_T_live)
        system = np.zeros(27, np.float64)
        rc2 = C.c_double()
        inliers, photometric = C.c_uint32(), C.c_uint32()
        self.lib.call("track_linearize_rgbd", self._h, _stream_handle(stream), C.byref(tp), C.byref(rp), level,
                      float(depth_scaling), lp, lpitch, lc, lcpitch, mp, mpitch, np_, npitch, mc, mcpitch,
                      T.ctypes.data_as(C.c_void_p), system.ctypes.data_as(C.c_void_p), C.byref(rc2), C.byref(inliers),
                      C.byref(photometric))
        return system, float(rc2.value), int(inliers.value), int(photometric.value)

    def relocalise(self, db: "KeyframeDatabase", depth, color, params: Optional[RelocParams] = None,
                   rgbd: Optional[TrackRGBDParams] = None, pp: Optional[PreprocessParams] = None, stream=None):
        """sm_relocalise: the pose of a frame the tracker lost (raw depth [H, W] uint16 and colour [H, W, 3] uint8 CUDA
        tensors at the handle's camera size), tracked against the cloud from the poses of `db`'s nearest keyframes in
        turn (params: the query and acceptance fields; None = the database's own). With `rgbd` the attempts track with
        colour (sm_track_frame_rgbd). Synchronous. Returns (pose [3, 4] float32, NaN when not relocalised,
        RelocResult)."""
        p = db.params if params is None else params
        pp = pp if pp is not None else PreprocessParams.defaults()
        self._check_raster("depth", depth, (self.height, self.width), torch.uint16)
        self._check_raster("color", color, (self.height, self.width, 3), torch.uint8)
        dp, dpitch = _raster(depth)
        cp, cpitch = _raster(color, 3)
        out = np.zeros(12, np.float32)
        result = RelocResult()
        self.lib.call("relocalise", self._h, db._h, _stream_handle(stream), C.byref(p), C.byref(pp),
                      C.byref(rgbd) if rgbd is not None else None, dp, dpitch, cp, cpitch,
                      out.ctypes.data_as(C.c_void_p), C.byref(result))
        return out.reshape(3, 4), result

    def triangulate(self, params: Optional[MeshParams] = None, stream=None):
        """sm_triangulate: the current cloud as a triangle mesh over its slots (include/surfel_b200.h gives the
        rules). Synchronous. Returns (triangles int32 CUDA tensor [T, 3] of slot indices, counter-clockwise about
        the owner's normal, MeshStats). Tries a capacity of 2 x surfels_size() first and retries once with the
        reported count."""
        p = MeshParams.defaults() if params is None else params
        handle = _stream_handle(stream)
        stats = MeshStats()
        capacity = max(2 * self.surfels_size(), 1)
        for attempt in range(2):
            out = torch.empty((capacity, 3), dtype=torch.int32, device="cuda")
            if isinstance(stream, torch.cuda.Stream):
                out.record_stream(stream)
            status = self.lib.fn["triangulate"](self._h, handle, C.byref(p), C.c_void_p(out.data_ptr()), capacity,
                                                C.byref(stats))
            if status == _lib.SM_ERR_CAPACITY and attempt == 0:
                capacity = max(int(stats.triangle_count), 1)
                continue
            if status != _lib.SM_OK:
                raise self.lib.error(status)
            return out[:int(stats.triangle_count)], stats
        raise AssertionError("unreachable")

    def mesh_update(self, params: Optional[MeshParams] = None, stream=None) -> MeshUpdateStats:
        """sm_mesh_update: brings the handle's persistent mesh up to date with the current cloud, rebuilding only
        the umbrellas a change can reach (include/surfel_b200.h gives the rules). Synchronous. Afterwards
        mesh_triangles("all") equals triangulate(params) on this state, and mesh_triangles("added" / "removed")
        are the triangles the update added and removed."""
        p = MeshParams.defaults() if params is None else params
        stats = MeshUpdateStats()
        self.lib.call("mesh_update", self._h, _stream_handle(stream), C.byref(p), C.byref(stats))
        return stats

    _MESH_LISTS = {"all": _lib.MESH_ALL, "added": _lib.MESH_ADDED, "removed": _lib.MESH_REMOVED}

    def mesh_triangles(self, which: str = "all", stream=None):
        """sm_mesh_read: one list of the last mesh_update() as an int32 CUDA tensor [T, 3] of slot indices, ordered
        by owner slot, then the owner's umbrella order. Asks for the count first (capacity 0), so a delta of a few
        triangles allocates only that much; retries once should the count change in between."""
        code = self._MESH_LISTS[which]
        handle = _stream_handle(stream)
        count = C.c_uint64()
        status = self.lib.fn["mesh_read"](self._h, handle, code, None, 0, C.byref(count))
        if status not in (_lib.SM_OK, _lib.SM_ERR_CAPACITY):
            raise self.lib.error(status)
        capacity = max(int(count.value), 1)
        for attempt in range(2):
            out = torch.empty((capacity, 3), dtype=torch.int32, device="cuda")
            if isinstance(stream, torch.cuda.Stream):
                out.record_stream(stream)
            status = self.lib.fn["mesh_read"](self._h, handle, code, C.c_void_p(out.data_ptr()), capacity,
                                              C.byref(count))
            if status == _lib.SM_ERR_CAPACITY and attempt == 0:
                capacity = max(int(count.value), 1)
                continue
            if status != _lib.SM_OK:
                raise self.lib.error(status)
            return out[:int(count.value)]
        raise AssertionError("unreachable")

    def fill_holes(self, triangles, params: Optional[HoleParams] = None, stream=None):
        """sm_mesh_fill_holes: the triangles that close the small boundary loops of `triangles` (an int32 CUDA
        tensor [T, 3] of slot indices, edge-manifold and consistently oriented, as triangulate() and
        mesh_triangles() return it; include/surfel_b200.h gives the rules). Synchronous. Returns (fill int32 CUDA
        tensor [F, 3], in the mesh's convention, to be appended to `triangles`; HoleStats). Asks for the count first
        (capacity 0), then writes."""
        p = HoleParams.defaults() if params is None else params
        _check_triangles(triangles)
        tri = triangles.contiguous()
        handle = _stream_handle(stream)
        stats = HoleStats()
        fn = self.lib.fn["mesh_fill_holes"]
        status = fn(self._h, handle, C.byref(p), C.c_void_p(tri.data_ptr()), len(tri), None, 0, C.byref(stats))
        if status not in (_lib.SM_OK, _lib.SM_ERR_CAPACITY):
            raise self.lib.error(status)
        capacity = max(int(stats.triangles_added), 1)
        out = torch.empty((capacity, 3), dtype=torch.int32, device="cuda")
        if isinstance(stream, torch.cuda.Stream):
            out.record_stream(stream)
        self.lib.call("mesh_fill_holes", self._h, handle, C.byref(p), C.c_void_p(tri.data_ptr()), len(tri),
                      C.c_void_p(out.data_ptr()), capacity, C.byref(stats))
        return out[:int(stats.triangles_added)], stats

    def simplify_mesh(self, triangles, params: Optional[SimplifyParams] = None, stream=None):
        """sm_mesh_simplify: `triangles` (an int32 CUDA tensor [T, 3] of slot indices, edge-manifold and consistently
        oriented, as triangulate() and fill_holes() give it) with slots removed by half-edge collapses, down to
        params.target_triangles or params.max_cost (include/surfel_b200.h gives the rules). Synchronous. Returns
        (int32 CUDA tensor [T', 3] over a subset of the slots, in the mesh's convention; SimplifyStats). The output
        is never longer than the input, so one call with capacity T suffices."""
        p = SimplifyParams.defaults() if params is None else params
        _check_triangles(triangles)
        tri = triangles.contiguous()
        out = torch.empty((max(len(tri), 1), 3), dtype=torch.int32, device="cuda")
        if isinstance(stream, torch.cuda.Stream):
            out.record_stream(stream)
        stats = SimplifyStats()
        self.lib.call("mesh_simplify", self._h, _stream_handle(stream), C.byref(p), C.c_void_p(tri.data_ptr()),
                      len(tri), C.c_void_p(out.data_ptr()), len(tri), C.byref(stats))
        return out[:int(stats.triangles_out)], stats

    def mesh_components(self, triangles, params: Optional[ComponentParams] = None, stream=None):
        """sm_mesh_components: the connected pieces of `triangles` (an int32 CUDA tensor [T, 3] of present slots, any
        list without repeated corners; two triangles are connected when they share an edge; include/surfel_b200.h
        gives the rules), and the triangles of the pieces that pass params (by default, pieces of at least 10
        triangles). Synchronous. Returns (kept int32 CUDA tensor [T', 3], the input's triangles in input order;
        labels int32 CUDA tensor [T], the number of each triangle's piece, pieces numbered by their first triangle;
        the piece table, a dict of CUDA tensors over the P pieces: "triangles" int64 [P], "area" float64 [P] (m^2),
        "lo" and "hi" float32 [P, 3] (smooth-position bounds), "first_triangle" int64 [P], "kept" bool [P];
        ComponentStats)."""
        p = ComponentParams.defaults() if params is None else params
        _check_triangles(triangles)
        tri = triangles.contiguous()
        T = len(tri)
        size = C.sizeof(MeshComponent)
        out = torch.empty((max(T, 1), 3), dtype=torch.int32, device="cuda")
        labels = torch.empty(max(T, 1), dtype=torch.int32, device="cuda")
        raw = torch.empty((max(T, 1), size), dtype=torch.uint8, device="cuda")
        if isinstance(stream, torch.cuda.Stream):
            for t in (out, labels, raw):
                t.record_stream(stream)
        stats = ComponentStats()
        self.lib.call("mesh_components", self._h, _stream_handle(stream), C.byref(p),
                      C.c_void_p(tri.data_ptr()) if T else None, T, C.c_void_p(out.data_ptr()), T,
                      C.c_void_p(labels.data_ptr()), C.c_void_p(raw.data_ptr()), T, C.byref(stats))
        raw = raw[:int(stats.components)]
        offset = {name: getattr(MeshComponent, name).offset for name, _ in MeshComponent._fields_}
        table = {"triangles": raw[:, offset["triangles"]:offset["triangles"] + 8].contiguous().view(torch.int64)[:, 0],
                 "area": raw[:, offset["area"]:offset["area"] + 8].contiguous().view(torch.float64)[:, 0],
                 "lo": raw[:, offset["lo"]:offset["lo"] + 12].contiguous().view(torch.float32),
                 "hi": raw[:, offset["hi"]:offset["hi"] + 12].contiguous().view(torch.float32),
                 "first_triangle": raw[:, offset["first_triangle"]:offset["first_triangle"] + 4].contiguous()
                 .view(torch.int32)[:, 0].to(torch.int64),
                 "kept": raw[:, offset["kept"]:offset["kept"] + 4].contiguous().view(torch.int32)[:, 0] != 0}
        return out[:int(stats.triangles_out)], labels[:T], table, stats

    def texture_mesh(self, triangles, views: Sequence[TextureView], params: Optional[TextureParams] = None,
                     stream=None):
        """sm_mesh_texture: a texture atlas for `triangles` (an int32 CUDA tensor [T, 3] of present slots, any list
        without repeated corners) from the colour images of `views` (TextureView, in the order their samples are
        summed; include/surfel_b200.h gives the rules). Synchronous. Lays the atlas out first (a query that writes
        nothing), then fills it. Returns (atlas uint8 CUDA tensor [H, W, 3], row 0 first; uv float32 CUDA tensor
        [T, 3, 2], (u, v) in [0, 1] per corner of each triangle in its listed order, v = 0 at row 0; TextureStats).
        Raises SurfelError (SM_ERR_CAPACITY) when the atlas would be wider than params.max_atlas_side: raise
        params.texel_size then."""
        p = TextureParams.defaults() if params is None else params
        _check_triangles(triangles)
        tri = triangles.contiguous()
        views = list(views)
        descs = (TextureViewDesc * max(len(views), 1))(*[v.desc() for v in views])
        handle = _stream_handle(stream)
        stats = TextureStats()
        fn = self.lib.fn["mesh_texture"]
        tri_ptr = C.c_void_p(tri.data_ptr()) if len(tri) else None
        status = fn(self._h, handle, C.byref(p), tri_ptr, len(tri), descs, len(views), None, 0, 0, 0, None,
                    C.byref(stats))
        if status == _lib.SM_OK:   # an empty list: an empty atlas
            return (torch.zeros((0, 0, 3), dtype=torch.uint8, device="cuda"),
                    torch.zeros((0, 3, 2), dtype=torch.float32, device="cuda"), stats)
        if status != _lib.SM_ERR_CAPACITY or stats.atlas_width > p.max_atlas_side:
            raise self.lib.error(status)
        W, H = int(stats.atlas_width), int(stats.atlas_height)
        atlas = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda")
        uv = torch.empty((len(tri), 3, 2), dtype=torch.float32, device="cuda")
        if isinstance(stream, torch.cuda.Stream):
            atlas.record_stream(stream)
            uv.record_stream(stream)
        self.lib.call("mesh_texture", self._h, handle, C.byref(p), tri_ptr, len(tri), descs, len(views),
                      C.c_void_p(atlas.data_ptr()), 3 * W, W, H, C.c_void_p(uv.data_ptr()), C.byref(stats))
        return atlas, uv, stats

    def export_vertices_host(self, stream=None):
        """sm_export_vertices into host arrays: positions [n, 3] float32 (NaN rows for merged slots), colours
        [n, 3] uint8, n = surfels_size()."""
        n = self.surfels_size()
        pos = torch.empty(max(3 * n, 3), dtype=torch.float32, device="cuda")
        col = torch.empty(max(3 * n, 3), dtype=torch.uint8, device="cuda")
        if n:
            self.ExportVertices(stream, pos, col)
        torch.cuda.synchronize()
        return pos[:3 * n].cpu().numpy().reshape(n, 3), col[:3 * n].cpu().numpy().reshape(n, 3)

    def save_mesh_obj(self, path, params: Optional[MeshParams] = None, stream=None,
                      holes: Optional[HoleParams] = None, simplify: Optional[SimplifyParams] = None,
                      texture: Optional[TextureParams] = None,
                      views: Optional[Sequence[TextureView]] = None,
                      components: Optional[ComponentParams] = None) -> MeshStats:
        """The reference's SaveMeshAsOBJ (main.cc:128-175): the non-merged slots in slot order with their colour,
        and the triangles of triangulate() over them (1-based, remapped to that order). With `holes`, the
        triangles of fill_holes(holes) follow the mesh's. With `components`, only the triangles of the pieces that
        mesh_components(components) keeps go on (after the fill, so floaters take no part of a simplification budget
        or of the atlas). With `simplify`, the mesh goes through simplify_mesh(simplify). With `components` or
        `simplify`, only the slots that are corners of the final triangles are written, in slot order.
        With `texture`, the final triangles are textured from `views` by texture_mesh(texture): the OBJ gets one
        texture coordinate per triangle corner and names the material of `path` with the suffix .mtl, whose
        diffuse map is the atlas written to `path` with the suffix .png."""
        tri, stats = self.triangulate(params, stream)
        if holes is not None:
            fill, _ = self.fill_holes(tri, holes, stream)
            tri = torch.cat([tri, fill])
        if components is not None:
            tri = self.mesh_components(tri, components, stream)[0]
        if simplify is not None:
            tri, _ = self.simplify_mesh(tri, simplify, stream)
        uvs, material = None, None
        if texture is not None:
            from pathlib import Path
            atlas, uv, _ = self.texture_mesh(tri, views or [], texture, stream)
            png, mtl = Path(path).with_suffix(".png"), Path(path).with_suffix(".mtl")
            image = atlas.cpu().numpy() if atlas.numel() else np.zeros((1, 1, 3), np.uint8)
            mesh_io.write_png(png, image)
            mesh_io.write_mtl(mtl, png.name)
            uvs, material = uv.cpu().numpy(), mtl.name
        positions, colors = self.export_vertices_host(stream)
        mesh_io.write_obj(path, positions, colors, tri.cpu().numpy(),
                          referenced_only=simplify is not None or components is not None, uvs=uvs, material=material)
        return stats

    def save_point_cloud_ply(self, path, stream=None) -> int:
        """The reference's SavePointCloudAsPLY (main.cc:180-203): position and normal of every non-merged slot,
        with its real colour (the reference writes white there). Returns the number of points written."""
        positions, colors = self.export_vertices_host(stream)
        rows, n, _ = self.dump_state(stream)
        return mesh_io.write_ply(path, positions, rows[8:11].T, colors)

    def ExportVertices(self, stream, position_buffer: torch.Tensor, color_buffer: torch.Tensor):
        """cuda_surfel_reconstruction.cc:405-410."""
        self.lib.call("export_vertices", self._h, _stream_handle(stream), C.c_void_p(position_buffer.data_ptr()),
                      C.c_void_p(color_buffer.data_ptr()))

    def GetTimings(self):
        """cuda_surfel_reconstruction.cc:412-429: (data_association, surfel_merging,
        measurement_blending, integration, neighbor_update, new_surfel_creation,
        regularization) in milliseconds."""
        out = (C.c_float * 7)()
        self.lib.call("get_timings", self._h, C.byref(out))
        return tuple(out)

    def enable_timings(self, enable=True):
        self.lib.call("enable_timings", self._h, 1 if enable else 0)

    def surfel_count(self) -> int:
        v = C.c_uint32()
        self.lib.call("surfel_count", self._h, C.byref(v))
        return v.value

    def surfels_size(self) -> int:
        v = C.c_uint32()
        self.lib.call("surfels_size", self._h, C.byref(v))
        return v.value

    # -- extras: fused pre-processing, state access, stream runner --------------------------
    def configure(self, key: str, value: float):
        """sm_configure: named tuning knobs (product only), e.g. "tiebreak_wave"."""
        self.lib.call("configure", self._h, key.encode(), float(value))

    def reset(self, stream=None):
        self.lib.call("reset", self._h, _stream_handle(stream))

    def preprocess(self, stream, params: PreprocessParams, raw_depth, other_depths, others_TR_reference, out_depth,
                   out_normals, out_radius):
        """The pre-processing call sequence of APP/main.cc:1015-1191 in one call."""
        K, ptrs, pitches, mats = _others_args(other_depths, others_TR_reference)
        assert K == params.outlier_filtering_frame_count
        rp, rpitch = _raster(raw_depth)
        op, opitch = _raster(out_depth)
        np_, npitch = _raster(out_normals, 2)
        radp, radpitch = _raster(out_radius)
        self.lib.call("preprocess", self._h, _stream_handle(stream), C.byref(params), rp, rpitch, ptrs, pitches,
                      mats.ctypes.data_as(C.c_void_p), op, opitch, np_, npitch, radp, radpitch)

    def dump_state(self, stream=None):
        """Returns (rows[25, n] float32 view of the SoA, surfels_size, merge_count)."""
        n = self.surfels_size()
        rows = np.zeros((_lib.ROW_COUNT, max(n, 1)), dtype=np.float32)
        size, merges = C.c_uint32(), C.c_uint32()
        self.lib.call("dump_state", self._h, _stream_handle(stream), rows.ctypes.data_as(C.c_void_p), rows.shape[1],
                      C.byref(size), C.byref(merges))
        assert size.value == n
        return rows[:, :n], n, merges.value

    def load_state(self, rows: np.ndarray, merge_count: int, stream=None):
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        assert rows.shape[0] == _lib.ROW_COUNT
        n = rows.shape[1]
        if n == 0:
            rows = np.zeros((_lib.ROW_COUNT, 1), dtype=np.float32)
        self.lib.call("load_state", self._h, _stream_handle(stream), rows.ctypes.data_as(C.c_void_p), rows.shape[1],
                      n, int(merge_count))

    def download_rasters(self, stream=None) -> dict:
        P = self.width * self.height
        out = {
            "supporting_surfels": np.empty(P, np.uint32), "supporting_surfel_counts": np.empty(P, np.uint32),
            "supporting_surfel_depth_sums": np.empty(P, np.float32), "conflicting_surfels": np.empty(P, np.uint32),
            "first_surfel_depth": np.empty(P, np.float32), "new_surfel_flag_vector": np.empty(P, np.uint8),
            "new_surfel_indices": np.empty(P, np.uint32),
        }
        self.lib.call("download_rasters", self._h, _stream_handle(stream),
                      *[v.ctypes.data_as(C.c_void_p) for v in out.values()])
        return {k: v.reshape(self.height, self.width) for k, v in out.items()}

    def stream_run(self, stream, depth, color, global_T_frame, frame_T_global, others_TR_reference,
                   pp: PreprocessParams, ip: IntegrateParams, first_frame: int, last_frame: int) -> StreamStats:
        """Frame loop of APP/main.cc:885-1223 over frames [first_frame, last_frame).

        depth [F,H,W] uint16 and color [F,H,W,3] uint8 are either CUDA tensors (device-resident
        stream) or pinned CPU tensors (uploaded frame by frame inside the call). H and W are the
        handle's size, or 2^L times it with configure("pyramid_level", L)."""
        on_host = not depth.is_cuda
        assert depth.is_contiguous() and color.is_contiguous() and color.is_cuda == depth.is_cuda
        if on_host:
            assert depth.is_pinned() and color.is_pinned(), "host frames must be in pinned memory"
        F = depth.shape[0]
        g = np.ascontiguousarray(np.asarray(global_T_frame, np.float32).reshape(F, 12))
        l = np.ascontiguousarray(np.asarray(frame_T_global, np.float32).reshape(F, 12))
        o = np.ascontiguousarray(np.asarray(others_TR_reference, np.float32).reshape(F, -1, 12))
        assert o.shape[1] == pp.outlier_filtering_frame_count
        H, W = depth.shape[1:3]
        assert tuple(color.shape[1:3]) == (H, W)
        desc = StreamDesc(W, H, F, 1 if on_host else 0, depth.data_ptr(), color.data_ptr(),
                          g.ctypes.data, l.ctypes.data, o.ctypes.data)
        stats = StreamStats()
        self.lib.call("stream_run", self._h, _stream_handle(stream), C.byref(desc), C.byref(pp), C.byref(ip),
                      int(first_frame), int(last_frame), C.byref(stats))
        return stats

    def compact(self, stream=None, return_map: bool = False):
        """sm_compact: removes the slots of merged surfels in place, keeping the order of the others. Returns
        CompactStats, or (CompactStats, old_to_new) with `return_map`: an int64 CUDA tensor of surfels_size()
        entries before the call, the new slot of each old one or -1 for a removed slot (remap_triangles applies it).
        Between the pushes of a session, call it through the session (StreamSession.compact), on its stream."""
        stats = CompactStats()
        if not return_map:
            self.lib.call("compact", self._h, _stream_handle(stream), None, 0, C.byref(stats))
            return stats
        n = self.surfels_size()
        out = torch.empty(max(n, 1), dtype=torch.int32, device="cuda")
        self.lib.call("compact", self._h, _stream_handle(stream), C.c_void_p(out.data_ptr()), n, C.byref(stats))
        old_to_new = out[:n].to(torch.int64) & 0xFFFFFFFF
        old_to_new[old_to_new == _lib.INVALID_SURFEL_INDEX] = -1
        return stats, old_to_new

    def session(self, pp: PreprocessParams, ip: IntegrateParams, frame_size, first_frame_index: int = 0,
                stream=None, compact_when_free_below: Optional[float] = None) -> "StreamSession":
        """An incremental session (sm_session_begin): the frame loop of APP/main.cc:885-1293 with frames pushed
        one at a time. `frame_size` = (width, height) of the sensor frames. Use as a context manager::

            with rec.session(pp, ip, (640, 480)) as s:
                for depth, color, g, l in frames:
                    s.push(depth, color, g, l)
            s.stats   # StreamStats of sm_session_end

        `compact_when_free_below` (a fraction of the surfel cap, default None = never): see StreamSession.
        """
        return StreamSession(self, pp, ip, frame_size, first_frame_index, stream, compact_when_free_below)


class KeyframeDatabase:
    """A keyframe database of random-fern codes (sm_keyframe_db_create), bound to the device and camera size of
    `rec`: add() stores frames that look new with their poses, query() finds the stored keyframes nearest to a frame,
    and CUDASurfelReconstruction.relocalise() restarts tracking from them. Frames are raw depth [H, W] uint16 and
    colour [H, W, 3] uint8 CUDA tensors at the handle's camera size."""

    def __init__(self, rec: CUDASurfelReconstruction, params: Optional[RelocParams] = None):
        self.lib = rec.lib
        self.params = RelocParams.defaults() if params is None else RelocParams.from_buffer_copy(params)
        self.width, self.height = rec.width, rec.height
        self.words = self.params.ferns // 8
        h = C.c_void_p()
        self.lib.call("keyframe_db_create", C.byref(h), rec._h, C.byref(self.params))
        self._h = h

    def close(self):
        if self._h:
            self.lib.fn["keyframe_db_destroy"](self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _frame(self, depth, color):
        for name, t, shape, dtype in (("depth", depth, (self.height, self.width), torch.uint16),
                                      ("color", color, (self.height, self.width, 3), torch.uint8)):
            if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape or t.dtype != dtype:
                raise ValueError(f"{name} must be a {dtype} tensor of shape {shape}")
        return (*_raster(depth), *_raster(color, 3))

    def __len__(self) -> int:
        n = C.c_uint32()
        self.lib.call("keyframe_db_count", self._h, C.byref(n))
        return int(n.value)

    def reset(self):
        """Forgets every keyframe (the fern tables stay)."""
        self.lib.call("keyframe_db_reset", self._h)

    def encode(self, depth, color, depth_scaling: float = 5000.0, stream=None) -> torch.Tensor:
        """sm_keyframe_db_encode: the frame's code, int32 CUDA tensor [ferns / 8] (the uint32 words' bits)."""
        out = torch.empty(self.words, dtype=torch.int32, device=depth.device)
        self.lib.call("keyframe_db_encode", self._h, _stream_handle(stream), *self._frame(depth, color),
                      float(depth_scaling), C.c_void_p(out.data_ptr()))
        return out

    def add(self, depth, color, global_T_frame, force: bool = False, depth_scaling: float = 5000.0, stream=None):
        """sm_keyframe_db_add: stores the frame as a keyframe if the database is empty, `force` is set, or it is far
        enough from every stored one. Synchronous. Returns (index, or -1 when not stored, full)."""
        g = _mat12(global_T_frame)
        index, full = C.c_int32(), C.c_int32()
        self.lib.call("keyframe_db_add", self._h, _stream_handle(stream), *self._frame(depth, color),
                      float(depth_scaling), g.ctypes.data_as(C.c_void_p), 1 if force else 0, C.byref(index),
                      C.byref(full))
        return int(index.value), bool(full.value)

    def query(self, depth, color, depth_scaling: float = 5000.0, stream=None):
        """sm_keyframe_db_query: the nearest keyframes in (distance, index) order within the query bound. Synchronous.
        Returns (indices int32 [found], distances uint32 [found])."""
        index = np.zeros(_lib.RELOC_MAX_CANDIDATES, np.int32)
        distance = np.zeros(_lib.RELOC_MAX_CANDIDATES, np.uint32)
        found = C.c_int32()
        self.lib.call("keyframe_db_query", self._h, _stream_handle(stream), *self._frame(depth, color),
                      float(depth_scaling), index.ctypes.data_as(C.c_void_p), distance.ctypes.data_as(C.c_void_p),
                      C.byref(found))
        return index[:found.value].copy(), distance[:found.value].copy()

    def pose(self, i: int) -> np.ndarray:
        """The [3, 4] float32 global_T_frame keyframe `i` was stored with."""
        out = np.zeros(12, np.float32)
        self.lib.call("keyframe_db_read", self._h, int(i), out.ctypes.data_as(C.c_void_p), None)
        return out.reshape(3, 4)

    def code(self, i: int) -> np.ndarray:
        """Keyframe `i`'s code, uint32 [ferns / 8]."""
        out = np.zeros(self.words, np.uint32)
        self.lib.call("keyframe_db_read", self._h, int(i), None, out.ctypes.data_as(C.c_void_p))
        return out


def _dtype_name(a) -> str:
    """'uint16', 'uint8', ... of a torch tensor or a numpy-convertible array."""
    if isinstance(a, torch.Tensor):
        return str(a.dtype).replace("torch.", "")
    return np.asarray(a).dtype.name


def _frame_arg(a, channels: int):
    """(pointer, pitch in bytes, on_host, keep-alive) of a depth [H, W] or colour [H, W, 3] frame: a CUDA tensor
    (row-pitched), or any CPU tensor / array (copied to a contiguous array if it is not row-pitched)."""
    if isinstance(a, torch.Tensor) and a.is_cuda:
        ptr, pitch = _raster(a, channels)
        return ptr, pitch, 0, a
    if isinstance(a, torch.Tensor):
        a = a.numpy()
    a = np.asarray(a)
    inner_ok = a.ndim == (2 if channels == 1 else 3) and a.strides[-1] == a.itemsize and (
        channels == 1 or a.strides[1] == channels * a.itemsize)
    if not inner_ok or a.strides[0] <= 0:
        a = np.ascontiguousarray(a)
    return C.c_void_p(a.ctypes.data), a.strides[0], 1, a


def remap_triangles(triangles: torch.Tensor, old_to_new: torch.Tensor) -> torch.Tensor:
    """A triangle list [T, 3] over the slots before sm_compact, over the slots after it (CUDASurfelReconstruction.
    compact(return_map=True)). A triangle with a removed corner is dropped; the others keep their order and
    corners. Lists from sm_triangulate or sm_mesh_fill_holes name present slots only, which sm_compact keeps."""
    tri = triangles.reshape(-1, 3).to(device=old_to_new.device, dtype=torch.int64)
    mapped = old_to_new[tri]
    return mapped[(mapped >= 0).all(dim=1)].to(triangles.dtype)


class StreamSession:
    """An open sm_session_begin on a CUDASurfelReconstruction (see CUDASurfelReconstruction.session).

    With `compact_when_free_below` = f (0 < f < 1), every push is followed by sm_compact when fewer than f x the
    surfel cap slots are free (surfels_size() > (1 - f) x cap): a long session is then bounded by the surfels it
    holds rather than by every surfel it created. The check costs a synchronisation per push. `compactions` holds
    the CompactStats of every compaction of the session, by policy or by compact()."""

    def __init__(self, rec: CUDASurfelReconstruction, pp: PreprocessParams, ip: IntegrateParams, frame_size,
                 first_frame_index: int = 0, stream=None, compact_when_free_below: Optional[float] = None):
        if compact_when_free_below is not None and not 0.0 < compact_when_free_below < 1.0:
            raise ValueError("compact_when_free_below must be a fraction of the surfel cap in (0, 1)")
        self.rec, self.pp, self.ip = rec, pp, ip
        self.width, self.height = (int(v) for v in frame_size)
        self.stream = _stream_handle(stream)
        self.stats: Optional[StreamStats] = None
        self.compact_when_free_below = compact_when_free_below
        self.compactions: list = []
        rec.lib.call("session_begin", rec._h, self.stream, C.byref(pp), C.byref(ip), self.width, self.height,
                     int(first_frame_index))
        self.open = True

    def push(self, depth, color, global_T_frame, frame_T_global) -> SessionStatus:
        """sm_session_push: depth [H, W] uint16 and colour [H, W, 3] uint8 as CUDA tensors or any CPU tensor /
        array (copied into pinned staging before the call returns), and the frame's two 3x4 poses."""
        if tuple(depth.shape[:2]) != (self.height, self.width) or tuple(color.shape[:2]) != (self.height, self.width):
            raise ValueError(f"frames must be {self.height} x {self.width}")
        if _dtype_name(depth) != "uint16" or _dtype_name(color) != "uint8" or len(color.shape) != 3 or color.shape[2] != 3:
            raise ValueError("depth must be uint16 [H, W] and colour uint8 [H, W, 3]")
        dp, dpitch, d_host, _keep_d = _frame_arg(depth, 1)
        cp, cpitch, c_host, _keep_c = _frame_arg(color, 3)
        if d_host != c_host:
            raise ValueError("depth and colour must both be CUDA tensors or both host memory")
        g = _mat12(global_T_frame)
        l = _mat12(frame_T_global)
        status = SessionStatus()
        self.rec.lib.call("session_push", self.rec._h, dp, dpitch, cp, cpitch, d_host, g.ctypes.data_as(C.c_void_p),
                          l.ctypes.data_as(C.c_void_p), C.byref(status))
        f = self.compact_when_free_below
        if f is not None and self.rec.surfels_size() > (1.0 - f) * self.rec.max_surfel_count:
            self.compact()
        return status

    def compact(self, return_map: bool = False):
        """sm_compact between two pushes, on the session's stream (CUDASurfelReconstruction.compact)."""
        result = self.rec.compact(self.stream, return_map)
        self.compactions.append(result[0] if return_map else result)
        return result

    def end(self) -> StreamStats:
        """sm_session_end: integrates what is left and returns the session's StreamStats."""
        if self.open:
            self.open = False
            stats = StreamStats()
            self.rec.lib.call("session_end", self.rec._h, C.byref(stats))
            self.stats = stats
        return self.stats

    def __enter__(self) -> "StreamSession":
        return self

    def __exit__(self, exc_type, exc, tb):
        if exc_type is None:
            self.end()
        elif self.open:   # an error inside the block: drain and close without masking it
            self.open = False
            self.rec.lib.fn["session_end"](self.rec._h, None)
        return False


def _to4(m) -> np.ndarray:
    return np.concatenate([np.asarray(m, np.float64).reshape(3, 4), [[0.0, 0.0, 0.0, 1.0]]], axis=0)


class TrackedSession:
    """A pose-free stream: every frame is tracked (sm_track_frame) and then pushed into a StreamSession with the pose
    it tracked. Only the first frame's camera-to-world pose is given. Frames are at the handle's camera size. With
    `rgbd` set, every frame is tracked with its own colour as well (sm_track_frame_rgbd), the first one included, so
    that its intensity is kept as the model of the second.

    Each frame after the first starts from a constant-velocity guess, T_{k-1} (T_{k-2}^-1 T_{k-1}). It is tracked
    against the previous frame until the session has integrated a frame, and against the cloud after that. A lost
    frame keeps its guess. `trajectory` holds the [3, 4] float32 poses pushed, `results` the TrackResults
    (TrackRGBDResults with `rgbd`)::

        with TrackedSession(rec, pp, ip, first_pose) as s:
            for depth, color in frames:
                s.push(depth, color)
        s.trajectory

    With `reloc` set, the session keeps a KeyframeDatabase (`database`): every frame tracked or relocalised against
    the cloud is offered to it (add()). A lost frame is relocalised (CUDASurfelReconstruction.relocalise, with colour
    when `rgbd` is set): if that succeeds it is pushed with the relocalised pose and the constant-velocity guess
    restarts from that pose; if not, the frame is held out of the session (not pushed, push() returns None) and the
    next frame tries again. `trajectory` stays indexed by frame, with NaN poses for held-out frames. `states` holds
    "tracked", "relocalised" or "lost" per frame (without `reloc` a "lost" frame is pushed with its guess, as
    above) and `reloc_results` the RelocResult of each relocalisation (None where none was tried).

    `compact_when_free_below` and compact() are StreamSession's: the merged slots are reclaimed between pushes."""

    def __init__(self, rec: CUDASurfelReconstruction, pp: PreprocessParams, ip: IntegrateParams, first_pose,
                 params: Optional[TrackParams] = None, first_frame_index: int = 0, stream=None,
                 rgbd: Optional[TrackRGBDParams] = None, reloc: Optional[RelocParams] = None,
                 compact_when_free_below: Optional[float] = None):
        self.rec, self.pp = rec, pp
        self.params = TrackParams.defaults() if params is None else params
        self.rgbd = rgbd
        self.reloc = reloc
        self.first_pose = np.asarray(first_pose, np.float32).reshape(3, 4)
        self.database = KeyframeDatabase(rec, reloc) if reloc is not None else None
        self.session = StreamSession(rec, pp, ip, (rec.width, rec.height), first_frame_index, stream,
                                     compact_when_free_below)
        self.trajectory: list = []
        self.results: list = []
        self.states: list = []
        self.reloc_results: list = []
        self.history: list = []   # the poses the constant-velocity guess extrapolates
        self.integrated = False

    def guess(self) -> np.ndarray:
        if len(self.history) < 2:
            return self.history[-1]
        a, b = _to4(self.history[-2]), _to4(self.history[-1])
        return (b @ np.linalg.inv(a) @ b)[:3].astype(np.float32)

    def push(self, depth, color) -> Optional[SessionStatus]:
        d = depth if isinstance(depth, torch.Tensor) and depth.is_cuda else torch.as_tensor(np.asarray(depth)).cuda()
        stream = self.session.stream
        c = None
        if self.rgbd is not None or self.reloc is not None:
            c = color if isinstance(color, torch.Tensor) and color.is_cuda else torch.as_tensor(np.asarray(color)).cuda()
        if self.rgbd is None:
            track = lambda *args: self.rec.track(d, *args)
        else:
            track = lambda guess, params, pp, source, stream: self.rec.track_rgbd(d, c, guess, params, self.rgbd, pp,
                                                                                  source, stream)
        if not self.history:
            # the first frame's view is kept as the model of the second: no Gauss-Newton steps, the given pose
            seed = TrackParams.from_buffer_copy(self.params)
            seed.levels = 1
            seed.iterations = (C.c_int32 * 4)(0, 0, 0, 0)
            pose, result = track(self.first_pose, seed, self.pp, "cloud", stream)
        else:
            pose, result = track(self.guess(), self.params, self.pp, "cloud" if self.integrated else "previous",
                                 stream)
        self.results.append(result)
        reloc_result = None
        state = "tracked" if (result.tracked if self.rgbd is None else result.depth.tracked) else "lost"
        if self.reloc is not None and self.history and state == "lost":
            pose, reloc_result = self.rec.relocalise(self.database, d, c, self.reloc, self.rgbd, self.pp, stream)
            state = "relocalised" if reloc_result.relocalised else "lost"
        self.states.append(state)
        self.reloc_results.append(reloc_result)
        self.trajectory.append(pose)
        if state == "lost" and self.reloc is not None:
            return None   # held out: not pushed, the next frame tries again from the same history
        if state == "relocalised":
            self.history = [pose]
        else:
            self.history.append(pose)
        if self.reloc is not None and (self.integrated or state == "relocalised"):
            self.database.add(d, c, pose, depth_scaling=self.pp.depth_scaling, stream=stream)
        status = self.session.push(depth, color, pose, invert_rigid(pose))
        self.integrated = status.last_integrated_frame >= 0
        return status

    def compact(self, return_map: bool = False):
        """sm_compact between two pushes (StreamSession.compact)."""
        return self.session.compact(return_map)

    def end(self) -> StreamStats:
        return self.session.end()

    def __enter__(self) -> "TrackedSession":
        return self

    def __exit__(self, exc_type, exc, tb):
        return self.session.__exit__(exc_type, exc, tb)


def outlier_filter_transforms(global_T_frame, frame_T_global, frame: int, other_count: int, depth_scaling: float,
                              lib: Optional[Library] = None) -> np.ndarray:
    """sm_outlier_filter_transforms: the [K, 3, 4] float32 transforms of reference frame `frame`
    (APP/main.cc:1039-1058) from [F, 3, 4] poses."""
    lib = lib or _lib.load_product()
    g = np.ascontiguousarray(np.asarray(global_T_frame, np.float32).reshape(-1, 12))
    l = np.ascontiguousarray(np.asarray(frame_T_global, np.float32).reshape(-1, 12))
    assert g.shape == l.shape
    out = np.zeros((int(other_count), 12), np.float32)
    lib.call("outlier_filter_transforms", int(other_count), float(depth_scaling), g.shape[0], g.ctypes.data_as(C.c_void_p),
             l.ctypes.data_as(C.c_void_p), int(frame), out.ctypes.data_as(C.c_void_p))
    return out.reshape(-1, 3, 4)


def stream_outlier_filter_transforms(global_T_frame, frame_T_global, other_count: int, depth_scaling: float,
                                     lib: Optional[Library] = None) -> np.ndarray:
    """[F, K, 3, 4] float32 for sm_stream_run / stream_run, by sm_outlier_filter_transforms; frames without K/2
    neighbours get identity (as synthetic.others_TR_reference)."""
    F = np.asarray(global_T_frame).reshape(-1, 12).shape[0]
    half = int(other_count) // 2
    out = np.tile(np.eye(4, dtype=np.float32)[:3][None, None], (F, int(other_count), 1, 1))
    for frame in range(half, F - half):
        out[frame] = outlier_filter_transforms(global_T_frame, frame_T_global, frame, other_count, depth_scaling, lib)
    return out
