"""ctypes loader for tests/mesh_render_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_render_mesh. The
library is compiled on first use into a temporary directory (keyed by the digest of its sources), so the repository
tree stays untouched."""
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
SOURCE = HERE / "mesh_render_walk.c"
SOURCES = (SOURCE, HERE / "render_walk.c")   # the first includes the second
DISK = 0x80000000
INVALID = 0xFFFFFFFF

_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(b"".join(p.read_bytes() for p in SOURCES)).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"mesh_render_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"libmesh_render_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the mesh render checker")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-o", str(tmp),
                            str(SOURCE), "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
        _lib.mrw_render.restype = None
        _lib.mrw_render.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int, C.c_int,
                                    C.c_int] + [C.c_float] * 6 + [C.c_void_p] * 7
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


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
    load().mrw_render(_p(rows), rows.shape[1], n, _p(tris), count, 1 if unmeshed_surfels else 0, int(width),
                      int(height), fx, fy, cx, cy, near, far, _p(T), _p(out["depth"]), _p(out["color"]),
                      _p(out["normal"]), _p(out["index"]), _p(keys), _p(st))
    if stats:
        return out, {"triangles": int(st[0]), "disks": int(st[1]), "marked": int(st[2])}
    return out
