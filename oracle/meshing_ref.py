"""ctypes loader for oracle/_ref/libmeshing_ref.so — TEST INFRASTRUCTURE.

The library is the reference's own CPU meshing (surfel_meshing.cc + octree.cc compiled unmodified by oracle/Makefile
against oracle/eigen_shim and oracle/libvis_stubs) behind oracle/meshing_driver.cc: BASELINE config 1 (random surfels
-> octree k-NN + Triangulate(), the pattern of the reference's test/test_triangulation.cc). Needs the reference sources
(oracle/Makefile: REF) at BUILD time only.
"""
from __future__ import annotations

import ctypes as C
import math
from pathlib import Path

import numpy as np

LIB_PATH = Path(__file__).resolve().parent / "_ref" / "libmeshing_ref.so"
_lib = None
_F = C.POINTER(C.c_float)
_U = C.POINTER(C.c_uint32)


def available() -> bool:
    return LIB_PATH.exists()


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(str(LIB_PATH))
        lib.smmesh_create.restype = C.c_void_p
        lib.smmesh_create.argtypes = [C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int]
        lib.smmesh_destroy.argtypes = [C.c_void_p]
        lib.smmesh_integrate.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, _F, _F, _F, _F, _F, _F, _F, _U]
        lib.smmesh_set_knn_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_int, _F, _U, C.POINTER(C.c_int32), _F]
        lib.smmesh_triangulate.argtypes = [C.c_void_p]
        lib.smmesh_check_remeshing.argtypes = [C.c_void_p]
        lib.smmesh_remesh_at.argtypes = [C.c_void_p, C.c_uint32, C.c_float]
        lib.smmesh_triangle_count.restype = C.c_uint64
        lib.smmesh_triangle_count.argtypes = [C.c_void_p]
        lib.smmesh_get_triangles.restype = C.c_uint64
        lib.smmesh_get_triangles.argtypes = [C.c_void_p, _U, C.c_uint64]
        lib.smmesh_meshing_states.argtypes = [C.c_void_p, C.POINTER(C.c_uint8), C.c_uint32]
        lib.smmesh_query_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        _lib = lib
    return _lib


class SurfelMeshing:
    """vis::SurfelMeshing with main.cc's defaults (main.cc:374-400, 481)."""

    MAX_NEIGHBOR_SEARCH_RANGE_INCREASE_FACTOR = 2.0

    def __init__(self, max_surfels_per_node=50, max_angle_between_normals_deg=90.0, min_triangle_angle_deg=10.0,
                 max_triangle_angle_deg=170.0, long_edge_tolerance_factor=1.5, regularization_frame_window_size=30):
        rad = math.pi / 180.0
        self._h = load().smmesh_create(max_surfels_per_node, max_angle_between_normals_deg * rad, min_triangle_angle_deg * rad,
                                       max_triangle_angle_deg * rad, self.MAX_NEIGHBOR_SEARCH_RANGE_INCREASE_FACTOR,
                                       long_edge_tolerance_factor, regularization_frame_window_size)
        self.count = 0

    def close(self):
        if self._h:
            load().smmesh_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def integrate(self, frame_index, x, y, z, radius_squared, nx, ny, nz, stamp):
        """IntegrateCUDABuffers on the eight CUDASurfelBuffersCPU arrays (follow with check_remeshing, triangulate)."""
        arrays = [np.ascontiguousarray(a, np.float32) for a in (x, y, z, radius_squared, nx, ny, nz)]
        stamp = np.ascontiguousarray(stamp, np.uint32)
        self.count = len(arrays[0])
        load().smmesh_integrate(self._h, int(frame_index), self.count, *[a.ctypes.data_as(_F) for a in arrays],
                                stamp.ctypes.data_as(_U))

    def set_knn_batch(self, d2, idx, count, batch_radius_squared):
        d2 = np.ascontiguousarray(d2, np.float32)
        idx = np.ascontiguousarray(idx, np.uint32)
        count = np.ascontiguousarray(count, np.int32)
        r2 = np.ascontiguousarray(batch_radius_squared, np.float32)
        load().smmesh_set_knn_batch(self._h, d2.shape[0], d2.shape[1], d2.ctypes.data_as(_F), idx.ctypes.data_as(_U),
                                    count.ctypes.data_as(C.POINTER(C.c_int32)), r2.ctypes.data_as(_F))

    def check_remeshing(self):
        load().smmesh_check_remeshing(self._h)

    def triangulate(self):
        load().smmesh_triangulate(self._h)

    def remesh_at(self, surfel_index, radius_factor_squared=4.0):
        load().smmesh_remesh_at(self._h, int(surfel_index), float(radius_factor_squared))

    def triangles(self):
        n = load().smmesh_triangle_count(self._h)
        out = np.zeros((max(n, 1), 3), np.uint32)
        got = load().smmesh_get_triangles(self._h, out.ctypes.data_as(_U), n)
        return out[:got]

    def meshing_states(self):
        out = np.zeros(self.count, np.uint8)
        load().smmesh_meshing_states(self._h, out.ctypes.data_as(C.POINTER(C.c_uint8)), self.count)
        return out

    def query_stats(self):
        served, fallback = C.c_uint64(), C.c_uint64()
        load().smmesh_query_stats(self._h, C.byref(served), C.byref(fallback))
        return served.value, fallback.value
