"""ctypes loader for tests/render_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_render_surfels."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from tests import cbuild
from tests.cbuild import ptr

SOURCE = Path(__file__).resolve().parent / "render_walk.c"


def load():
    return cbuild.library(SOURCE, cbuild.WALK_FLAGS, {
        "rw_render": (None, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_int] + [C.c_float] * 6 +
                      [C.c_void_p] * 6)})


def render(rows, view_T_global, width, height, fx, fy, cx, cy, near, far) -> dict:
    """sm_render_surfels on a [25, n] float32 state (rows 3-5 = smooth positions, as sm_dump_state returns them).
    Returns depth [H, W] float32, color [H, W, 3] uint8, normal [H, W, 3] float32, index [H, W] uint32."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    if n == 0:
        rows = np.zeros((rows.shape[0], 1), np.float32)
    T = np.ascontiguousarray(np.asarray(view_T_global, np.float32).reshape(-1)[:12])
    out = {"depth": np.empty((height, width), np.float32), "color": np.empty((height, width, 3), np.uint8),
           "normal": np.empty((height, width, 3), np.float32), "index": np.empty((height, width), np.uint32)}
    keys = np.empty(max(width * height, 1), np.uint64)
    load().rw_render(ptr(rows), rows.shape[1], n, int(width), int(height), fx, fy, cx, cy, near, far, ptr(T),
                     ptr(out["depth"]), ptr(out["color"]), ptr(out["normal"]), ptr(out["index"]), ptr(keys))
    return out
