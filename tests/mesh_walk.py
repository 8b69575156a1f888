"""ctypes loader for tests/mesh_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_triangulate, plus the
hand-built clouds and the mesh invariants the host and GPU tests share."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from surfelmeshing_b200 import _lib as L
from tests import cbuild
from tests import knn_cases
from tests.cbuild import ptr

SOURCE = Path(__file__).resolve().parent / "mesh_walk.c"
U = L.MESH_MAX_UMBRELLA


def load():
    return cbuild.library(SOURCE, cbuild.WALK_FLAGS, {
        "mw_triangulate": (C.c_uint64, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p])})


def triangulate(rows, params=None):
    """sm_triangulate on a [25, n] float32 state (rows 3-5 = smooth positions, as sm_dump_state returns them).
    Returns (triangles uint32 [T, 3], stats dict, umbrella counts [n])."""
    p = params or L.MeshParams.defaults()
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    if n == 0:
        rows = np.zeros((rows.shape[0], 1), np.float32)
    umbrella = np.zeros(max(n, 1) * U * 2, np.uint32)
    counts = np.zeros(max(n, 1), np.uint32)
    stats = np.zeros(4, np.uint64)
    lib = load()
    args = (ptr(rows), rows.shape[1], n, p.neighbor_radius_factor, p.max_angle_between_normals_deg,
            p.max_triangle_angle_deg, U, ptr(umbrella), ptr(counts))
    total = lib.mw_triangulate(*args, None, 0, ptr(stats))
    tri = np.zeros((max(total, 1), 3), np.uint32)
    lib.mw_triangulate(*args, ptr(tri), total, ptr(stats))
    names = ("triangle_count", "vertices_meshed", "boundary_edges", "umbrella_overflows")
    return tri[:total], {k: int(v) for k, v in zip(names, stats)}, counts[:n]


# ---- hand-built clouds ---------------------------------------------------------------------------------------

def make_rows(positions, normals, radius_squared):
    """[25, n] float32 state: rows 0-2 and 3-5 the positions, 7 radius^2, 8-10 the normals, no links."""
    positions = np.asarray(positions, np.float32).reshape(-1, 3)
    n = len(positions)
    rows = np.zeros((L.ROW_COUNT, n), np.float32)
    rows.view(np.uint32)[19:23] = 0xFFFFFFFF
    rows[0:3] = positions.T
    rows[3:6] = positions.T
    rows[6] = 1.0
    rows[7] = np.broadcast_to(np.asarray(radius_squared, np.float32), (n,))
    rows[8:11] = np.broadcast_to(np.asarray(normals, np.float32).reshape(-1, 3), (n, 3)).T
    rows.view(np.uint32)[24] = (np.arange(n, dtype=np.uint32) * 2654435761) & 0xFFFFFF
    return rows


def grid(side, spacing):
    u, v = np.meshgrid(np.arange(side), np.arange(side), indexing="ij")
    return u.ravel() * spacing, v.ravel() * spacing


def jittered_plane(side=30, spacing=0.01, seed=1):
    rng = np.random.default_rng(seed)
    x, y = grid(side, spacing)
    x = x + rng.uniform(-0.25, 0.25, x.size) * spacing
    y = y + rng.uniform(-0.25, 0.25, y.size) * spacing
    pos = np.stack([x, y, np.full(x.size, 1.0)], 1)
    perm = rng.permutation(len(pos))   # slot order is creation order, not spatial order
    return make_rows(pos[perm], (0, 0, 1), (1.3 * spacing) ** 2)


def pixel_grid(side=24, spacing=2.0 ** -7):
    """Exact grid points on z = 1 with normal +z: every unit square is a cocircular quad."""
    x, y = grid(side, spacing)
    return make_rows(np.stack([x, y, np.full(x.size, 1.0)], 1), (0, 0, 1), (1.3 * spacing) ** 2)


def sphere(n=2000, radius=0.5):
    k = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * k / n)
    theta = np.pi * (1 + 5 ** 0.5) * k
    d = np.stack([np.cos(theta) * np.sin(phi), np.sin(theta) * np.sin(phi), np.cos(phi)], 1)
    spacing = np.sqrt(4 * np.pi * radius ** 2 / n)
    return make_rows(d * radius, d, (1.2 * spacing) ** 2)


def crossing_planes(degrees, side=24, spacing=0.01):
    """Two planes through the x axis, degrees apart, each with its own normal."""
    x, y = grid(side, spacing)
    y = y - y.mean()
    a = np.radians(degrees)
    first = np.stack([x, y, np.zeros_like(x)], 1)
    second = np.stack([x, y * np.cos(a), y * np.sin(a)], 1)
    normals = np.concatenate([np.tile([0.0, 0.0, 1.0], (len(x), 1)),
                              np.tile([0.0, -np.sin(a), np.cos(a)], (len(x), 1))])
    pos = np.concatenate([first, second]) + np.array([0.0, 0.0, 1.0])
    return make_rows(pos, normals, (1.3 * spacing) ** 2)


def meshing_cloud(kind, n=3000, seed=5):
    c = knn_cases.meshing_cloud(n, seed, kind)
    pos = np.stack([c["x"], c["y"], c["z"]], 1)
    return make_rows(pos, np.stack([c["nx"], c["ny"], c["nz"]], 1), c["radius_squared"])


def with_duplicates(seed=2):
    rows = jittered_plane(side=16, seed=seed)
    n = rows.shape[1]
    rng = np.random.default_rng(seed)
    src = rng.choice(n, 20, replace=False)
    return np.concatenate([rows, rows[:, src]], 1)


def with_merged(seed=3):
    rows = jittered_plane(side=16, seed=seed)
    rng = np.random.default_rng(seed)
    rows[7, rng.choice(rows.shape[1], 30, replace=False)] *= -1
    return rows


def with_flipped_normals(seed=4):
    rows = jittered_plane(side=16, seed=seed)
    rng = np.random.default_rng(seed)
    rows[8:11, rng.choice(rows.shape[1], 20, replace=False)] *= -1
    return rows


def golden_f7():
    from tests.util import GOLDEN_DIR, load_npz_xz
    return load_npz_xz(GOLDEN_DIR / "golden_320x240_f7.npz.xz")["f7_state"]


CASES = {
    "jittered_plane": jittered_plane,
    "pixel_grid": pixel_grid,
    "sphere": sphere,
    "planes_90": lambda: crossing_planes(90),
    "planes_30": lambda: crossing_planes(30),
    "sheet": lambda: meshing_cloud("sheet"),
    "cube": lambda: meshing_cloud("cube"),
    "duplicates": with_duplicates,
    "merged": with_merged,
    "flipped_normals": with_flipped_normals,
    "empty": lambda: make_rows(np.zeros((0, 3)), (0, 0, 1), 1e-4),
    "single": lambda: make_rows(np.array([[0.0, 0.0, 1.0]]), (0, 0, 1), 1e-4),
}


# ---- invariants ----------------------------------------------------------------------------------------------

def check_invariants(rows, tri):
    """Indices are present slots, no repeated corner or triangle, every directed edge at most once, each triangle
    counter-clockwise about its first corner's normal (the owner), owners ascending. Returns the directed-edge set."""
    tri = np.asarray(tri, np.int64).reshape(-1, 3)
    if len(tri) == 0:
        return set()
    n = rows.shape[1]
    assert (tri >= 0).all() and (tri < n).all()
    assert (rows[7, tri] > 0).all(), "a corner is not a present slot"
    assert (tri[:, 0] != tri[:, 1]).all() and (tri[:, 1] != tri[:, 2]).all() and (tri[:, 0] != tri[:, 2]).all()
    assert (tri[:, 0] < tri[:, 1]).all() and (tri[:, 0] < tri[:, 2]).all(), "not written by the smallest index"
    assert (np.diff(tri[:, 0]) >= 0).all(), "owners not ascending"
    canon = np.sort(tri, 1)
    assert len(np.unique(canon, axis=0)) == len(tri), "a triangle appears twice"
    edges = np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [2, 0]]])
    assert len(np.unique(edges, axis=0)) == len(edges), "a directed edge appears twice"
    p = rows[3:6].T.astype(np.float64)
    g = np.cross(p[tri[:, 1]] - p[tri[:, 0]], p[tri[:, 2]] - p[tri[:, 0]])
    assert (np.einsum("ij,ij->i", g, rows[8:11].T[tri[:, 0]].astype(np.float64)) > 0).all(), "orientation"
    return {tuple(e) for e in edges.tolist()}


def topology(tri):
    """(V, E, F, boundary edges, boundary loops) of the triangles' own vertices."""
    tri = np.asarray(tri, np.int64).reshape(-1, 3)
    if len(tri) == 0:
        return 0, 0, 0, 0, 0
    directed = [tuple(e) for e in np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [2, 0]]]).tolist()]
    present = set(directed)
    boundary = [e for e in directed if (e[1], e[0]) not in present]
    edge_count = len({tuple(sorted(e)) for e in directed})
    nxt = {a: b for a, b in boundary}
    loops, seen = 0, set()
    for a in nxt:
        if a in seen:
            continue
        loops += 1
        while a not in seen:
            seen.add(a)
            a = nxt.get(a, a)
    return len(np.unique(tri)), edge_count, len(tri), len(boundary), loops


def area(rows, tri):
    p = rows[3:6].T.astype(np.float64)
    tri = np.asarray(tri, np.int64).reshape(-1, 3)
    return 0.5 * np.linalg.norm(np.cross(p[tri[:, 1]] - p[tri[:, 0]], p[tri[:, 2]] - p[tri[:, 0]]), axis=1).sum()
