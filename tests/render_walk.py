"""ctypes loader for tests/render_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_render_surfels. The
library is compiled on first use into a temporary directory (keyed by the source's digest), so the repository tree
stays untouched."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

SOURCE = Path(__file__).resolve().parent / "render_walk.c"

_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(SOURCE.read_bytes()).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"render_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"librender_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the render checker")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-o", str(tmp),
                            str(SOURCE), "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
        _lib.rw_render.restype = None
        _lib.rw_render.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_int] + [C.c_float] * 6 + \
            [C.c_void_p] * 6
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


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
    load().rw_render(_p(rows), rows.shape[1], n, int(width), int(height), fx, fy, cx, cy, near, far, _p(T),
                     _p(out["depth"]), _p(out["color"]), _p(out["normal"]), _p(out["index"]), _p(keys))
    return out
