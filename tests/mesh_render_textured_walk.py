"""ctypes loader for tests/mesh_render_textured_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of
sm_render_mesh_textured, built on tests/mesh_render_walk.c's. The library is compiled on first use into a temporary
directory (keyed by the digest of its sources), so the repository tree stays untouched."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
SOURCE = HERE / "mesh_render_textured_walk.c"
SOURCES = (SOURCE, HERE / "mesh_render_walk.c", HERE / "render_walk.c")   # each includes the next

_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(b"".join(p.read_bytes() for p in SOURCES)).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"mesh_render_textured_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"libmesh_render_textured_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the textured mesh render checker")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-o", str(tmp),
                            str(SOURCE), "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
        _lib.mrtw_render.restype = None
        _lib.mrtw_render.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int, C.c_int,
                                     C.c_int] + [C.c_float] * 6 + [C.c_void_p] * 3 + [C.c_int, C.c_int] + \
            [C.c_void_p] * 6
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


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
    load().mrtw_render(_p(rows), rows.shape[1], n, _p(tris), count, 1 if unmeshed_surfels else 0, int(width),
                       int(height), fx, fy, cx, cy, near, far, _p(T), _p(uv), _p(atlas) if atlas.size else None,
                       atlas.shape[1], atlas.shape[0], _p(out["depth"]), _p(out["color"]), _p(out["normal"]),
                       _p(out["index"]), _p(keys), None)
    return out
