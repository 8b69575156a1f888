"""ctypes loader for tests/simplify_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of sm_mesh_simplify, and
the hand-built meshes the host and GPU tests share. The library is compiled on first use into a temporary directory
(keyed by the source's digest), so the repository tree stays untouched."""
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
from tests import hole_walk as HW
from tests import mesh_walk as M

SOURCE = Path(__file__).resolve().parent / "simplify_walk.c"
STAT_NAMES = [f for f, _ in L.SimplifyStats._fields_]
ERRORS = {-1: "bad corner", -2: "repeated corner", -3: "duplicate edge"}

_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(SOURCE.read_bytes()).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"simplify_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"libsimplify_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the simplification checker")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-o", str(tmp),
                            str(SOURCE), "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
        _lib.sw_simplify.restype = C.c_int64
        _lib.sw_simplify.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64,
                                     C.POINTER(L.SimplifyParams), C.c_void_p, C.c_uint64, C.POINTER(L.SimplifyStats),
                                     C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class InvalidMesh(ValueError):
    pass


class OrderDependent(AssertionError):
    pass


def stats_dict(stats):
    return {k: getattr(stats, k) for k in STAT_NAMES if k != "reserved"}


def simplify(rows, tri, params=None, log=False):
    """sm_mesh_simplify on a [25, n] float32 state (rows 3-5 = smooth positions) and a [T, 3] triangle list.
    Returns (triangles uint32 [T', 3], stats dict), plus with log=True a dict: "rounds" = [(selected, applied)] per
    round and "last_selected" = the keys the last applied round selected, ascending. Raises InvalidMesh for an input
    the call rejects and OrderDependent if the two application orders of a round disagree."""
    p = params or L.SimplifyParams.defaults()
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    if n == 0:
        rows = np.zeros((rows.shape[0], 1), np.float32)
    tri = np.ascontiguousarray(np.asarray(tri, np.uint32).reshape(-1, 3))
    count = len(tri)
    out = np.zeros((max(count, 1), 3), np.uint32)
    stats = L.SimplifyStats()
    round_log = np.zeros((max(p.max_rounds, 1), 2), np.uint64)
    last = np.zeros(max(count, 1), np.uint64)
    last_count = C.c_uint64()
    total = load().sw_simplify(_p(rows), rows.shape[1], n, _p(tri) if count else None, count, C.byref(p), _p(out),
                               count, C.byref(stats), _p(round_log), _p(last), C.byref(last_count))
    if total == -4:
        raise OrderDependent("a round's collapses depend on their order")
    if total < 0:
        raise InvalidMesh(ERRORS[total])
    result = (out[:total], stats_dict(stats))
    if log:
        return result + ({"rounds": [tuple(int(x) for x in r) for r in round_log[:stats.rounds]],
                          "last_selected": last[:last_count.value].copy()},)
    return result


def unbounded(**overrides):
    """Parameters with no bound but the geometry: no cost limit, no normal gate, no angle limit, every round."""
    values = dict(max_cost=float("inf"), max_angle_between_normals_deg=180.0, max_triangle_angle_deg=180.0,
                  max_rounds=L.SIMPLIFY_MAX_ROUNDS)
    values.update(overrides)
    return L.SimplifyParams.defaults(**values)


# ---- hand-built meshes ---------------------------------------------------------------------------------------

def outward(positions, tri, centre):
    """tri with each triangle wound counter-clockwise seen from outside (away from `centre`)."""
    p = np.asarray(positions, np.float64)
    out = []
    for a, b, c in tri:
        g = np.cross(p[b] - p[a], p[c] - p[a])
        out.append((a, b, c) if g @ (p[[a, b, c]].mean(0) - centre) > 0 else (a, c, b))
    return HW.canonical(out)


# A slightly irregular octahedron (6 slots, 8 triangles) with normals pointing away from its centre.
OCTAHEDRON_POSITIONS = [[1.0, 0.05, 0.02], [-0.9, 0.1, -0.05], [0.03, 1.1, 0.04], [-0.06, -0.95, 0.08],
                        [0.07, -0.02, 1.05], [0.02, 0.04, -1.2]]


def octahedron():
    pos = np.asarray(OCTAHEDRON_POSITIONS)
    rows = M.make_rows(pos, pos / np.linalg.norm(pos, axis=1, keepdims=True), 1e-2)
    tri = [(a, b, c) for a in (0, 1) for b in (2, 3) for c in (4, 5)]
    return rows, outward(pos, tri, np.zeros(3))


def neck(rings=(1.0, 0.15, 1.0), heights=(-1.0, 0.0, 1.0), apex=2.0):
    """A closed hourglass: a bottom apex, three rings of three slots (the middle one a thin neck) and a top apex,
    with normals pointing away from the axis (the apexes along it). Collapsing two neck slots onto each other would
    pinch the surface into two spheres that touch."""
    pos = [[0.0, 0.0, -apex]]
    nrm = [[0.0, 0.0, -1.0]]
    for r, z in zip(rings, heights):
        for k in range(3):
            a = 2 * np.pi * k / 3 + (0.3 if r < 0.5 else 0.0)
            pos.append([r * np.cos(a), r * np.sin(a), z])
            nrm.append([np.cos(a), np.sin(a), 0.0])
    pos.append([0.0, 0.0, apex])
    nrm.append([0.0, 0.0, 1.0])
    tri = [(0, 1 + k, 1 + (k + 1) % 3) for k in range(3)]
    for ring in range(2):
        lo, hi = 1 + 3 * ring, 4 + 3 * ring
        for k in range(3):
            k1 = (k + 1) % 3
            tri += [(lo + k, lo + k1, hi + k), (lo + k1, hi + k1, hi + k)]
    tri += [(7 + k, 7 + (k + 1) % 3, 10) for k in range(3)]
    pos = np.asarray(pos)
    return M.make_rows(pos, nrm, 1e-2), outward(pos, tri, np.zeros(3))


def hub(spokes=40):
    """A flat disk on z = 1: slot 0 in the middle with `spokes` neighbours (slots 1..spokes on a circle of radius 1),
    and an outer circle of radius 2 (the next `spokes` slots), the band between the circles split into triangles.
    Every cost is 0, so a ring slot's best neighbour is its smallest valid one: the hub, were its valence in range."""
    a = 2 * np.pi * np.arange(spokes) / spokes
    inner = np.stack([np.cos(a), np.sin(a), np.ones(spokes)], 1)
    outer = np.stack([2 * np.cos(a + np.pi / spokes), 2 * np.sin(a + np.pi / spokes), np.ones(spokes)], 1)
    pos = np.concatenate([[[0.0, 0.0, 1.0]], inner, outer])
    tri = []
    for k in range(spokes):
        k1 = (k + 1) % spokes
        i, i1, o, o1 = 1 + k, 1 + k1, 1 + spokes + k, 1 + spokes + k1
        tri += [(0, i, i1), (i, o, i1), (i1, o, o1)]
    rows = M.make_rows(pos, (0, 0, 1), 1e-2)
    return rows, HW.canonical(tri)


def link_case():
    """A closed surface of 7 slots on which only the link condition, rule S3 (a), stops a collapse. Slot 0 is the
    centre of a flat square fan on z = 0 (ring 1, 2, 3, 4, normals +z); below it, two slots (5, 6, normals -z) close
    the surface with the edge 1-3 running under the fan. So N(0) and N(1) share 2, 4 and also 3. The collapse 0 -> 1
    costs 0, keeps the valences in range, moves the triangles (1, 2, 3) and (1, 3, 4), which face their corner
    normals, and repeats no triangle; it would put the directed edge 1 -> 3 in two triangles."""
    pos = [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0],
           [0.0, -0.5, -0.5], [0.0, 0.5, -0.5]]
    normals = [[0.0, 0.0, 1.0]] * 5 + [[0.0, 0.0, -1.0]] * 2
    tri = [(0, 1, 2), (0, 2, 3), (0, 3, 4), (0, 4, 1),
           (1, 4, 5), (4, 3, 5), (3, 1, 5), (1, 3, 6), (3, 2, 6), (2, 1, 6)]
    return M.make_rows(pos, normals, 1e-2), HW.canonical(tri)


def repeat_case():
    """A tetrahedron on which only rule S3 (c)'s repeated triangle stops a collapse: every normal is +z, so the
    triangle that collapsing the apex (slot 0) onto a base corner moves, the base (1, 3, 2) wound the other way,
    faces all three of its corner normals. The link condition holds (every slot has degree 3)."""
    pos = [[0.1, 0.05, 1.0], [0.0, 0.0, 0.0], [1.0, 0.1, 0.0], [0.2, 1.0, 0.0]]
    tri = [(0, 1, 2), (0, 2, 3), (0, 3, 1), (1, 3, 2)]
    return M.make_rows(pos, (0.0, 0.0, 1.0), 1e-2), HW.canonical(tri)


def meshed(rows):
    """The sm_triangulate mesh of a cloud (mesh_walk's restatement) with the fill of its holes (hole_walk's)."""
    tri, _, _ = M.triangulate(rows)
    fill, _ = HW.fill_holes(rows, tri)
    return np.concatenate([tri, fill]).astype(np.uint32)


def mesh_cases():
    """name -> (rows, triangles): the hand-built meshes, and the restated meshes of mesh_walk clouds."""
    cases = {"octahedron": octahedron(), "neck": neck(), "hub": hub()}
    for name in ("pixel_grid", "jittered_plane", "sphere", "planes_90", "sheet", "cube"):
        rows = M.CASES[name]()
        cases[name] = (rows, meshed(rows))
    return cases
