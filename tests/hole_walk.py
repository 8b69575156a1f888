"""ctypes loader for tests/hole_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_mesh_fill_holes, and
the hand-built meshes the host and GPU tests share. The library is compiled on first use into a temporary
directory (keyed by the source's digest), so the repository tree stays untouched."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

from surfelmeshing_b200 import _lib as L
from tests import mesh_walk as M

SOURCE = Path(__file__).resolve().parent / "hole_walk.c"
STAT_NAMES = [f for f, _ in L.HoleStats._fields_]
ERRORS = {-1: "bad corner", -2: "repeated corner", -3: "duplicate edge"}

_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(SOURCE.read_bytes()).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"hole_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"libhole_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the hole-filling checker")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-o", str(tmp),
                            str(SOURCE), "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
        _lib.hw_fill_holes.restype = C.c_int64
        _lib.hw_fill_holes.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int, C.c_float,
                                       C.c_float, C.c_void_p, C.c_uint64, C.c_void_p]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class InvalidMesh(ValueError):
    pass


def fill_holes(rows, tri, params=None):
    """sm_mesh_fill_holes on a [25, n] float32 state (rows 3-5 = smooth positions) and a [T, 3] triangle list.
    Returns (fill uint32 [F, 3], stats dict); raises InvalidMesh for an input the call rejects."""
    p = params or L.HoleParams.defaults()
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    if n == 0:
        rows = np.zeros((rows.shape[0], 1), np.float32)
    tri = np.ascontiguousarray(np.asarray(tri, np.uint32).reshape(-1, 3))
    stats = np.zeros(7, np.uint64)
    lib = load()
    args = (_p(rows), rows.shape[1], n, _p(tri) if len(tri) else None, len(tri), p.max_hole_edges,
            p.max_angle_between_normals_deg, p.max_triangle_angle_deg)
    total = lib.hw_fill_holes(*args, None, 0, _p(stats))
    if total < 0:
        raise InvalidMesh(ERRORS[total])
    fill = np.zeros((max(total, 1), 3), np.uint32)
    lib.hw_fill_holes(*args, _p(fill), total, _p(stats))
    return fill[:total], {k: int(v) for k, v in zip(STAT_NAMES, stats)}


# ---- hand-built meshes ---------------------------------------------------------------------------------------

SIDE_8 = 8


def grid_mesh(side):
    """The pixel grid of mesh_walk (side x side exact points on z = 1, normal +z) with every square split along
    its (0, 0)-(1, 1) diagonal, counter-clockwise about +z, in the mesh's convention. Slot of (i, j) = i * side + j
    (x = i, y = j)."""
    rows = M.pixel_grid(side)
    tri = []
    for i in range(side - 1):
        for j in range(side - 1):
            a, b, c, d = i * side + j, (i + 1) * side + j, (i + 1) * side + j + 1, i * side + j + 1
            tri += [(a, b, c), (a, c, d)]
    return rows, canonical(tri)


def canonical(tri):
    """Each triangle rotated to start at its smallest slot."""
    out = []
    for t in tri:
        r = int(np.argmin(t))
        out.append(tuple(t[r:]) + tuple(t[:r]))
    return np.asarray(out, np.uint32).reshape(-1, 3)


def without(tri, corners):
    """The triangles of `tri` that have none of `corners` as a corner."""
    tri = np.asarray(tri, np.uint32).reshape(-1, 3)
    return tri[~np.isin(tri, list(corners)).any(1)]


def covering(tri, slots):
    """The triangles whose three corners all lie in `slots`."""
    tri = np.asarray(tri, np.uint32).reshape(-1, 3)
    return tri[np.isin(tri, list(slots)).all(1)]


def without_triangles(tri, drop):
    tri = np.asarray(tri, np.uint32).reshape(-1, 3)
    drop = {tuple(t) for t in canonical(drop).tolist()}
    return tri[[tuple(t) not in drop for t in tri.tolist()]]


def square_hole(side, i, j):
    """Both triangles of the square with lower-left corner (i, j)."""
    a, b, c, d = i * side + j, (i + 1) * side + j, (i + 1) * side + j + 1, i * side + j + 1
    return canonical([(a, b, c), (a, c, d)])


def tilted_corner_case(degrees=45.0):
    """grid_mesh(8) with the square (2, 2) removed and the normal of its corner (3, 3) tilted by `degrees` about the
    x axis: the corner's pairs pass a normal gate wider than `degrees` and fail a narrower one."""
    rows, tri = grid_mesh(SIDE_8)
    t = np.radians(degrees)
    rows[8:11, 3 * SIDE_8 + 3] = (0.0, -np.sin(t), np.cos(t))
    return rows, without_triangles(tri, square_hole(SIDE_8, 2, 2))


# A non-planar quad loop (0, 1, 2, 3) whose input is a reversed pyramid over slot 4, so both diagonals are free:
# the smaller split, along 0-2, has an angle above 120 degrees, so a limit of 120 takes the split along 1-3.
ANGLE_POSITIONS = [[0.42, -0.28, 0.17], [0.83, 0.09, -0.15], [0.74, 1.09, -0.12], [-0.07, 1.34, 0.13],
                   [0.5, 0.5, -1.0]]


def angle_case():
    rows = M.make_rows(ANGLE_POSITIONS, (0, 0, 1), 1e-4)
    return rows, canonical([(4, 1, 0), (4, 2, 1), (4, 3, 2), (4, 0, 3)])


# Two loops that propose the same diagonal: a hexagon A = (0, 1, 2, 3, 4, 5) and a quad B = (0, 6, 3, 7) that
# share the pinch vertices 0 and 3. The input is A's and B's reversed caps (A's with the diagonals 1-5, 1-4, 2-4,
# B's with 6-7) and closed two-triangle pillows over the slots 8-10 that make 0-4, 1-3 and 2-5 input edges, so the
# only triangulations left are A: 0-2, 0-3, 3-5 and B: 0-3. Positions and normals are free in 3D (found by a
# seeded search, rounded to two decimals): each loop alone is filled, together both are dropped by rule H6.
CONFLICT_POSITIONS = [[0.0, 0.0, 0.0], [1.77, 0.0, 0.54], [-1.71, 0.99, -0.16], [0.34, -0.59, 0.62],
                      [-1.48, -1.38, 1.18], [0.0, 1.4, 0.73], [0.68, -1.08, -0.27], [1.08, -0.66, 0.06],
                      [5.23, 5.89, 5.17], [5.59, 5.87, 5.91], [5.62, 5.1, 5.01]]
CONFLICT_NORMALS = [[-0.57, -0.1, 0.82], [-0.28, -0.33, 0.9], [0.08, 0.29, 0.95], [-0.41, 0.68, -0.6],
                    [-0.29, 0.0, -0.96], [-0.88, -0.13, -0.45], [-0.85, -0.53, -0.04], [0.44, 0.76, 0.48],
                    [0.0, 0.0, 1.0], [0.0, 0.0, 1.0], [0.0, 0.0, 1.0]]


def conflict_case():
    """(rows, A's input alone, B's input alone, both together)."""
    rows = M.make_rows(CONFLICT_POSITIONS, CONFLICT_NORMALS, 1e-4)
    a = canonical([(0, 5, 1), (1, 5, 4), (1, 4, 2), (2, 4, 3),
                   (0, 4, 8), (4, 0, 8), (1, 3, 9), (3, 1, 9), (2, 5, 10), (5, 2, 10)])
    b = canonical([(0, 7, 6), (6, 7, 3)])
    return rows, a, b, np.concatenate([a, b])


def check_union(rows, tri, fill):
    """Mesh and fill together: every directed edge at most once, every fill triangle counter-clockwise about all
    three corner normals, written from its smallest slot. Returns topology() of the union."""
    tri = np.asarray(tri, np.int64).reshape(-1, 3)
    fill = np.asarray(fill, np.int64).reshape(-1, 3)
    both = np.concatenate([tri, fill])
    edges = np.concatenate([both[:, [0, 1]], both[:, [1, 2]], both[:, [2, 0]]])
    assert len(np.unique(edges, axis=0)) == len(edges), "a directed edge appears twice"
    if len(fill):
        assert (fill[:, 0] < fill[:, 1]).all() and (fill[:, 0] < fill[:, 2]).all()
        p = rows[3:6].T.astype(np.float64)
        g = np.cross(p[fill[:, 1]] - p[fill[:, 0]], p[fill[:, 2]] - p[fill[:, 0]])
        nrm = rows[8:11].T.astype(np.float64)
        for c in range(3):
            assert (np.einsum("ij,ij->i", g, nrm[fill[:, c]]) > 0).all(), "orientation"
    return M.topology(both)
