"""ctypes loader for tests/mesh_render_textured_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of
sm_render_mesh_textured, built on tests/mesh_render_walk.c's."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from tests import cbuild
from tests.cbuild import ptr

SOURCE = Path(__file__).resolve().parent / "mesh_render_textured_walk.c"


def load():
    return cbuild.library(SOURCE, cbuild.WALK_FLAGS, {
        "mrtw_render": (None, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int] +
                        [C.c_float] * 6 + [C.c_void_p] * 3 + [C.c_int, C.c_int] + [C.c_void_p] * 6)})


def render_textured(rows, triangles, texture, view_T_global, width, height, fx, fy, cx, cy, near, far,
                    unmeshed_surfels=True):
    """sm_render_mesh_textured on a [25, n] float32 state (rows 3-5 = smooth positions) and a [T, 3] list of slot
    indices, with texture = (atlas uint8 [H, W, 3], uv float32 [T, 3, 2]) as texture_mesh() returns them. Returns
    the dict of mesh_render_walk.render(): depth, color, normal, index."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    if n == 0:
        rows = np.zeros((rows.shape[0], 1), np.float32)
    tris = np.ascontiguousarray(np.asarray(triangles).reshape(-1, 3).astype(np.int64).astype(np.uint32))
    count = tris.shape[0]
    atlas = np.ascontiguousarray(texture[0], np.uint8)
    uv = np.ascontiguousarray(texture[1], np.float32).reshape(-1, 6)
    assert atlas.ndim == 3 and atlas.shape[2] == 3 and len(uv) == count
    if count == 0:
        tris, uv = np.zeros((1, 3), np.uint32), np.zeros((1, 6), np.float32)
    T = np.ascontiguousarray(np.asarray(view_T_global, np.float32).reshape(-1)[:12])
    out = {"depth": np.empty((height, width), np.float32), "color": np.empty((height, width, 3), np.uint8),
           "normal": np.empty((height, width, 3), np.float32), "index": np.empty((height, width), np.uint32)}
    keys = np.empty(max(width * height, 1), np.uint64)
    load().mrtw_render(ptr(rows), rows.shape[1], n, ptr(tris), count, 1 if unmeshed_surfels else 0, int(width),
                       int(height), fx, fy, cx, cy, near, far, ptr(T), ptr(uv), ptr(atlas) if atlas.size else None,
                       atlas.shape[1], atlas.shape[0], ptr(out["depth"]), ptr(out["color"]), ptr(out["normal"]),
                       ptr(out["index"]), ptr(keys), None)
    return out
