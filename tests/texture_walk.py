"""ctypes loader for tests/texture_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_mesh_texture, and the
hand-built scenes of the texture tests. The library is compiled on first use into a temporary directory (keyed by the
digest of its sources), so the repository tree stays untouched."""
from __future__ import annotations

import ctypes as C
import hashlib
import math
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

from surfelmeshing_b200._lib import TextureParams
from tests import mesh_walk as M

HERE = Path(__file__).resolve().parent
SOURCE = HERE / "texture_walk.c"
SOURCES = (SOURCE, HERE / "mesh_render_walk.c", HERE / "render_walk.c")   # each includes the next

_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(b"".join(p.read_bytes() for p in SOURCES)).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"texture_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"libtexture_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the texture checker")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-o", str(tmp),
                            str(SOURCE), "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
        _lib.txw_texture.restype = C.c_uint32
        _lib.txw_texture.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_float, C.c_float,
                                     C.c_float, C.c_int] + [C.c_void_p] * 7
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


STATS = ("triangles", "atlas_width", "atlas_height", "texels", "texels_seen", "texels_fallback", "tiles_clamped",
         "views_used")


def stats_dict(s) -> dict:
    return {k: int(getattr(s, k)) for k in STATS}


def cos_max(params) -> float:
    return float(np.float32(math.cos(float(params.max_view_angle_deg) * (math.pi / 180.0))))


class View:
    """A host view: camera dict (width, height, fx, fy, cx, cy), view_T_global [3, 4], colour uint8 [H, W, 3]."""

    def __init__(self, cam, T, color, near=0.1, far=100.0):
        self.cam, self.T = dict(cam), np.asarray(T, np.float32).reshape(3, 4)
        self.color = np.ascontiguousarray(color, np.uint8)
        self.near, self.far = float(near), float(far)
        assert self.color.shape == (cam["height"], cam["width"], 3)


def texture(rows, triangles, views, params=None, layout_only=False):
    """sm_mesh_texture on a [25, n] float32 state (rows 3-5 = smooth positions) and a [T, 3] list of slot indices.
    Returns (atlas uint8 [H, W, 3], uv float32 [T, 3, 2], stats dict); (None, None, stats) when the layout is wider
    than params.max_atlas_side or with layout_only. Raises ValueError for a list that breaks X1."""
    p = params or TextureParams.defaults()
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    tris = np.ascontiguousarray(np.asarray(triangles).reshape(-1, 3).astype(np.int64).astype(np.uint32))
    count = len(tris)
    if count == 0:
        tris = np.zeros((1, 3), np.uint32)
    V = len(views)
    size = np.array([[v.cam["width"], v.cam["height"]] for v in views] or [[1, 1]], np.int32)
    cam = np.array([[v.cam["fx"], v.cam["fy"], v.cam["cx"], v.cam["cy"], v.near, v.far] for v in views]
                   or [[1] * 6], np.float32)
    T = np.ascontiguousarray(np.array([v.T for v in views] or [np.zeros((3, 4))], np.float32))
    colors = (C.c_void_p * max(V, 1))(*[v.color.ctypes.data for v in views])
    st = np.zeros(8, np.uint64)
    lib = load()
    args = (_p(rows), rows.shape[1], n, _p(tris), count, float(p.texel_size), cos_max(p), float(p.depth_tolerance),
            V, _p(size), _p(cam), _p(T), C.cast(colors, C.c_void_p))
    errors = lib.txw_texture(*args, None, None, _p(st))
    if errors:
        raise ValueError(f"input error bits {errors}")
    stats = dict(zip(STATS, (int(x) for x in st)))
    if layout_only or stats["atlas_width"] > p.max_atlas_side:
        return None, None, stats
    W, H = stats["atlas_width"], stats["atlas_height"]
    atlas = np.zeros((max(H, 1), max(W, 1), 3), np.uint8)
    uv = np.zeros((max(count, 1), 3, 2), np.float32)
    lib.txw_texture(*args, _p(atlas), _p(uv), _p(st))
    return atlas[:H, :W], uv[:count], dict(zip(STATS, (int(x) for x in st)))


# ---- hand-built scenes ----------------------------------------------------------------------------------------

CAM = dict(width=96, height=80, fx=80.0, fy=80.0, cx=48.0, cy=40.0)


def quad_rows(z=1.0, half=0.3, grid=4, color=(200, 100, 50), offset=(0.0, 0.0)):
    """A (grid + 1)^2-vertex square at depth z facing the camera (normals -z), split into 2 grid^2 triangles wound
    counter-clockwise seen from the camera at the origin looking down +z. Returns (rows, triangles)."""
    xs = np.linspace(-half, half, grid + 1)
    pts = [(offset[0] + x, offset[1] + y, z) for y in xs for x in xs]
    rows = M.make_rows(pts, (0.0, 0.0, -1.0), (half / grid) ** 2)
    rgb = np.uint32(color[0] | (color[1] << 8) | (color[2] << 16))
    rows[24] = np.full(len(pts), rgb, np.uint32).view(np.float32)
    tris = []
    for j in range(grid):
        for i in range(grid):
            a, b, c, d = j * (grid + 1) + i, j * (grid + 1) + i + 1, (j + 1) * (grid + 1) + i, (j + 1) * (grid + 1) + i + 1
            tris += [(a, c, b), (b, c, d)]
    return rows, np.array(tris, np.int64)


def stack(*parts):
    """Concatenates (rows, triangles) pairs into one state, renumbering the triangles."""
    rows = np.concatenate([r for r, _ in parts], axis=1)
    out, base = [], 0
    for r, t in parts:
        out.append(np.asarray(t) + base)
        base += r.shape[1]
    return rows, np.concatenate(out)


def identity():
    return np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def look_from(eye, target=(0.0, 0.0, 1.0), up=(0.0, -1.0, 0.0)):
    """view_T_global of a camera at `eye` looking at `target` (y down in the image, as the identity camera)."""
    eye, target, up = (np.asarray(v, np.float64) for v in (eye, target, up))
    z = (target - eye) / np.linalg.norm(target - eye)
    x = np.cross(z, up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])   # rows: camera axes in world
    return np.hstack([R, (-R @ eye)[:, None]]).astype(np.float32)


def solid(cam, rgb):
    return np.broadcast_to(np.array(rgb, np.uint8), (cam["height"], cam["width"], 3)).copy()


def ramp(cam):
    """Red rises with x (2 per pixel), green with y (3 per pixel), blue constant."""
    H, W = cam["height"], cam["width"]
    img = np.zeros((H, W, 3), np.uint8)
    img[..., 0] = (2 * np.arange(W))[None, :]
    img[..., 1] = (3 * np.arange(H))[:, None]
    img[..., 2] = 77
    return img
