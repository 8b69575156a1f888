"""ctypes loader for tests/mesh_render_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_render_mesh."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from tests import cbuild
from tests.cbuild import ptr

SOURCE = Path(__file__).resolve().parent / "mesh_render_walk.c"
DISK = 0x80000000
INVALID = 0xFFFFFFFF


def load():
    return cbuild.library(SOURCE, cbuild.WALK_FLAGS, {
        "mrw_render": (None, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int] +
                       [C.c_float] * 6 + [C.c_void_p] * 7)})


def render(rows, triangles, view_T_global, width, height, fx, fy, cx, cy, near, far, unmeshed_surfels=True,
           stats=False):
    """sm_render_mesh on a [25, n] float32 state (rows 3-5 = smooth positions, as sm_dump_state returns them) and a
    [T, 3] list of slot indices. Returns depth [H, W] float32, color [H, W, 3] uint8, normal [H, W, 3] float32,
    index [H, W] uint32; with stats=True also {"triangles": drawn (covering a pixel centre), "disks": unmeshed
    slots inside [near, far], "marked": slots named by a T1-valid triangle}."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    if n == 0:
        rows = np.zeros((rows.shape[0], 1), np.float32)
    tris = np.ascontiguousarray(np.asarray(triangles).reshape(-1, 3).astype(np.int64).astype(np.uint32))
    if tris.size == 0:
        tris = np.zeros((1, 3), np.uint32)
        count = 0
    else:
        count = tris.shape[0]
    T = np.ascontiguousarray(np.asarray(view_T_global, np.float32).reshape(-1)[:12])
    out = {"depth": np.empty((height, width), np.float32), "color": np.empty((height, width, 3), np.uint8),
           "normal": np.empty((height, width, 3), np.float32), "index": np.empty((height, width), np.uint32)}
    keys = np.empty(max(width * height, 1), np.uint64)
    st = np.zeros(3, np.uint64)
    load().mrw_render(ptr(rows), rows.shape[1], n, ptr(tris), count, 1 if unmeshed_surfels else 0, int(width),
                      int(height), fx, fy, cx, cy, near, far, ptr(T), ptr(out["depth"]), ptr(out["color"]),
                      ptr(out["normal"]), ptr(out["index"]), ptr(keys), ptr(st))
    if stats:
        return out, {"triangles": int(st[0]), "disks": int(st[1]), "marked": int(st[2])}
    return out
