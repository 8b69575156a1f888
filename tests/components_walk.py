"""ctypes loader for tests/components_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_mesh_components,
and the hand-built meshes the host and GPU tests share."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from surfelmeshing_b200 import _lib as L
from tests import cbuild
from tests import mesh_walk as M
from tests import simplify_walk as SW
from tests.cbuild import ptr

SOURCE = Path(__file__).resolve().parent / "components_walk.c"
STATS = [f for f, _ in L.ComponentStats._fields_]
ERRORS = {-1: "bad corner", -2: "repeated corner"}
# sm_mesh_component as a numpy record
TABLE_DTYPE = np.dtype({"names": ["triangles", "area", "lo", "hi", "first_triangle", "kept"],
                        "formats": ["<u8", "<f8", ("<f4", 3), ("<f4", 3), "<u4", "<i4"],
                        "offsets": [getattr(L.MeshComponent, f).offset for f, _ in L.MeshComponent._fields_],
                        "itemsize": C.sizeof(L.MeshComponent)})


def load():
    return cbuild.library(SOURCE, cbuild.WALK_FLAGS, {
        "cw_components": (C.c_int64, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64,
                                      C.POINTER(L.ComponentParams), C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.POINTER(L.ComponentStats)])})


class InvalidMesh(ValueError):
    pass


def stats_dict(stats) -> dict:
    return {k: getattr(stats, k) for k in STATS}


def components(rows, tri, params=None):
    """sm_mesh_components on a [25, n] float32 state (rows 3-5 = smooth positions) and a [T, 3] triangle list.
    Returns (kept triangles uint32 [T', 3], labels int32 [T], table TABLE_DTYPE [P], stats dict). Raises InvalidMesh
    for a list that breaks C1."""
    p = params or L.ComponentParams.defaults()
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    if n == 0:
        rows = np.zeros((rows.shape[0], 1), np.float32)
    tri = np.ascontiguousarray(np.asarray(tri, np.int64).reshape(-1, 3).astype(np.uint32))
    count = len(tri)
    out = np.zeros((max(count, 1), 3), np.uint32)
    labels = np.zeros(max(count, 1), np.int32)
    table = np.zeros(max(count, 1), TABLE_DTYPE)
    stats = L.ComponentStats()
    total = load().cw_components(ptr(rows), rows.shape[1], n, ptr(tri) if count else None, count, C.byref(p), ptr(out),
                                 ptr(labels), ptr(table), C.byref(stats))
    if total < 0:
        raise InvalidMesh(ERRORS[total])
    return out[:total], labels[:count], table[:stats.components].copy(), stats_dict(stats)


# ---- hand-built meshes ---------------------------------------------------------------------------------------

def strip(origin, quads=3, size=0.1, normal_axis=2):
    """A strip of `quads` squares (2 triangles each) from `origin` along x, in the plane normal to `normal_axis`:
    (positions [2 (quads + 1), 3], triangles over them)."""
    pos = []
    for i in range(quads + 1):
        for j in range(2):
            p = [i * size, j * size, 0.0]
            if normal_axis == 1:
                p = [p[0], 0.0, p[1]]
            pos.append(np.asarray(origin, np.float64) + p)
    tri = []
    for i in range(quads):
        a, b, c, d = 2 * i, 2 * i + 1, 2 * i + 2, 2 * i + 3
        tri += [(a, c, b), (b, c, d)]
    return np.asarray(pos), np.asarray(tri)


def touching_planes():
    """Two fans of 6 triangles each, one on z = 1 and one on y = 0, that share only slot 0: 2 pieces."""
    ring = [(np.cos(a), np.sin(a)) for a in np.linspace(0, 2 * np.pi, 7)[:-1]]
    pos = [[0.0, 0.0, 1.0]] + [[0.2 * x, 0.2 * y + 0.3, 1.0] for x, y in ring]
    pos[0] = [0.0, 0.1, 1.0]
    pos += [[0.2 * x, 0.0, 1.0 + 0.2 * y - 0.3] for x, y in ring]
    # fan 1 around slot 1 (its ring 2..6 and slot 0 as its first ring slot), fan 2 around slot 7 likewise
    tri = [(1, 0, 2), (1, 2, 3), (1, 3, 4), (1, 4, 5), (1, 5, 6), (1, 6, 0),
           (7, 0, 8), (7, 8, 9), (7, 9, 10), (7, 10, 11), (7, 11, 12), (7, 12, 0)]
    return M.make_rows(pos, (0.0, 0.0, 1.0), 1e-2), np.asarray(tri)


def fin():
    """Three triangles on one edge {0, 1} (a non-manifold edge, windings mixed), and a fourth that meets only the
    third at an edge: 1 piece."""
    pos = [[0.0, 0.0, 1.0], [0.1, 0.0, 1.0], [0.05, 0.1, 1.0], [0.05, -0.1, 1.0], [0.05, 0.0, 1.1], [0.1, 0.0, 1.2]]
    tri = [(0, 1, 2), (1, 0, 3), (0, 1, 4), (4, 1, 5)]
    return M.make_rows(pos, (0.0, 0.0, 1.0), 1e-2), np.asarray(tri)


def islands():
    """An isolated triangle between two strips, a second isolated triangle last, and strips of 4 and 6 squares whose
    areas tie with each other's halves: pieces of 1, 8, 1, 12, 8 triangles, the two 8s equal in area (Q ties)."""
    parts, tri, offset = [], [], 0

    def add(pos, t):
        nonlocal offset
        parts.append(pos)
        tri.extend((np.asarray(t) + offset).tolist())
        offset += len(pos)
    single = np.array([[0.0, 0.0, 2.0], [0.125, 0.0, 2.0], [0.0, 0.125, 2.0]])
    add(single, [(0, 1, 2)])
    add(*strip((1.0, 0.0, 2.0), quads=4, size=0.125))
    add(single + [0.0, 1.0, 0.0], [(0, 1, 2)])
    add(*strip((1.0, 1.0, 2.0), quads=6, size=0.125))
    add(*strip((1.0, 2.0, 2.0), quads=4, size=0.125))
    pos = np.concatenate(parts)
    return M.make_rows(pos, (0.0, 0.0, 1.0), 1e-2), np.asarray(tri)


def shuffled(rows, tri, seed=7):
    """The same mesh with its triangle order and corner rotations permuted."""
    rng = np.random.default_rng(seed)
    t = np.asarray(tri)[rng.permutation(len(tri))]
    r = rng.integers(0, 3, len(t))
    return rows, np.stack([np.roll(x, k) for x, k in zip(t, r)]) if len(t) else t


def mesh_cases():
    """name -> (rows, triangles): the hand-built meshes, the restated meshes of mesh_walk clouds (with their fill),
    and a shuffled copy of two of them."""
    cases = {"touching_planes": touching_planes(), "fin": fin(), "islands": islands()}
    for name in ("pixel_grid", "jittered_plane", "sphere", "planes_90", "planes_30", "sheet", "cube", "duplicates",
                 "merged", "flipped_normals", "single", "empty"):
        rows = M.CASES[name]()
        cases[name] = (rows, SW.meshed(rows) if rows.shape[1] else np.zeros((0, 3), np.uint32))
    cases["sheet_shuffled"] = shuffled(*cases["sheet"])
    cases["islands_shuffled"] = shuffled(*cases["islands"], seed=3)
    return cases
