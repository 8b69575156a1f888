"""ctypes loader for oracle/_ref/liboctree_ref.so — TEST INFRASTRUCTURE.

The library is the reference's own CPU octree (applications/surfel_meshing/src/surfel_meshing/octree.cc, compiled
unmodified by oracle/Makefile against oracle/eigen_shim) behind the C entry points of oracle/octree_driver.cc, plus
a restatement of the brute-force checker of the reference's octree test (test/test_octree.cc:116-149). It needs
the reference sources (oracle/Makefile: REF) at BUILD time only.
"""
from __future__ import annotations

import ctypes as C
import time
from pathlib import Path

import numpy as np

LIB_PATH = Path(__file__).resolve().parent / "_ref" / "liboctree_ref.so"

_lib = None
_F = C.POINTER(C.c_float)
_U = C.POINTER(C.c_uint32)
_B = C.POINTER(C.c_uint8)
_I = C.POINTER(C.c_int32)


def available() -> bool:
    return LIB_PATH.exists()


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(str(LIB_PATH))
        lib.smoct_create.restype = C.c_void_p
        lib.smoct_create.argtypes = [C.c_int, C.c_uint32, _F, _F, _F, _F, _B]
        lib.smoct_destroy.argtypes = [C.c_void_p]
        lib.smoct_query_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint32, _F, _F, _F, _F, C.c_int, _F, _U, _I]
        lib.smoct_brute_force.restype = C.c_int
        lib.smoct_brute_force.argtypes = [C.c_uint32, _F, _F, _F, _B, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float,
                                          C.c_float, C.c_int, _F, _U]
        _lib = lib
    return _lib


def _f(a):
    return a.ctypes.data_as(_F) if a is not None else None


def _b(a):
    return a.ctypes.data_as(_B) if a is not None else None


class Octree:
    """CompressedOctree over (x, y, z) with optional per-point meshing state (255 = not inserted)."""

    def __init__(self, x, y, z, state=None, radius_squared=None, max_surfels_per_node: int = 50):
        self.x, self.y, self.z = [np.ascontiguousarray(a, np.float32) for a in (x, y, z)]
        self.state = None if state is None else np.ascontiguousarray(state, np.uint8)
        r2 = None if radius_squared is None else np.ascontiguousarray(radius_squared, np.float32)
        self._h = load().smoct_create(max_surfels_per_node, len(self.x), _f(self.x), _f(self.y), _f(self.z), _f(r2),
                                      _b(self.state))

    def close(self):
        if self._h:
            load().smoct_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def query(self, qx, qy, qz, radius_squared, max_result_count, include_completed=True, include_free=True):
        """FindNearestSurfelsWithinRadius<include_completed, include_free>, one query after the other on one
        thread (the meshing thread's pattern). Returns (d2 [Q, k], idx [Q, k], counts [Q], seconds)."""
        qx, qy, qz, r2 = [np.ascontiguousarray(a, np.float32) for a in (qx, qy, qz, radius_squared)]
        q, k = len(qx), int(max_result_count)
        d2 = np.full((q, k), np.inf, np.float32)
        idx = np.full((q, k), 0xFFFFFFFF, np.uint32)
        cnt = np.zeros(q, np.int32)
        t0 = time.perf_counter()
        load().smoct_query_batch(self._h, int(include_completed), int(include_free), q, _f(qx), _f(qy), _f(qz), _f(r2), k,
                                 _f(d2), idx.ctypes.data_as(_U), cnt.ctypes.data_as(_I))
        seconds = time.perf_counter() - t0
        for j in range(q):   # entries past the count are scratch in the reference; give them the product's fill
            d2[j, cnt[j]:] = np.inf
            idx[j, cnt[j]:] = 0xFFFFFFFF
        return d2, idx, cnt, seconds


def brute_force(x, y, z, state, qx, qy, qz, radius_squared, max_result_count, include_completed=True, include_free=True):
    """test_octree.cc:116-149 with the state filter and (distance, index) order; same return layout as Octree.query."""
    x, y, z = [np.ascontiguousarray(a, np.float32) for a in (x, y, z)]
    state = None if state is None else np.ascontiguousarray(state, np.uint8)
    q, k = len(qx), int(max_result_count)
    d2 = np.full((q, k), np.inf, np.float32)
    idx = np.full((q, k), 0xFFFFFFFF, np.uint32)
    cnt = np.zeros(q, np.int32)
    bd = np.zeros(k, np.float32)
    bi = np.zeros(k, np.uint32)
    lib = load()
    for j in range(q):
        c = lib.smoct_brute_force(len(x), _f(x), _f(y), _f(z), _b(state), int(include_completed), int(include_free),
                                  float(qx[j]), float(qy[j]), float(qz[j]), float(radius_squared[j]), k, _f(bd),
                                  bi.ctypes.data_as(_U))
        cnt[j] = c
        d2[j, :c] = bd[:c]
        idx[j, :c] = bi[:c]
    return d2, idx, cnt


def canonical_ties(d2, idx, cnt):
    """Orders runs of equal distance by index (the octree leaves them in traversal order) — only INSIDE the returned
    set; a tie that straddles the cap cannot be repaired this way and is reported by `tie_at_cap`."""
    d2, idx = d2.copy(), idx.copy()
    for j in range(len(cnt)):
        c = int(cnt[j])
        order = np.lexsort((idx[j, :c], d2[j, :c]))
        d2[j, :c], idx[j, :c] = d2[j, :c][order], idx[j, :c][order]
    return d2, idx
