"""TEST INFRASTRUCTURE: a numpy restatement of sm_mesh_update's rules (include/surfel_b200.h) on top of the plain-C
restatement of sm_triangulate (tests/mesh_walk.c). It computes the sets C, A and R between two states, the exact
umbrella and per-owner share of every slot in each state, and the mesh an update assembles from them: the
previous owners' triangles outside R, the new ones inside R."""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

from surfelmeshing_b200 import _lib as L
from tests import mesh_walk as M
from tests.cbuild import ptr

SNAPSHOT_ROWS = (3, 4, 5, 7, 8, 9, 10)   # smooth x y z, radius^2, normal x y z
WIDE = 64                                # an umbrella cap no slot reaches: the exact umbrella, overflow or not


def walk(rows, params=None, cap=M.U):
    """mw_triangulate with umbrella cap `cap`: (triangles [T, 3], stats dict, umbrellas [n, cap, 2], lengths [n])."""
    p = params or L.MeshParams.defaults()
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    n = rows.shape[1]
    store = rows if n else np.zeros((rows.shape[0], 1), np.float32)
    umbrella = np.zeros((max(n, 1), cap, 2), np.uint32)
    counts = np.zeros(max(n, 1), np.uint32)
    stats = np.zeros(4, np.uint64)
    lib = M.load()
    args = (ptr(store), store.shape[1], n, p.neighbor_radius_factor, p.max_angle_between_normals_deg,
            p.max_triangle_angle_deg, cap, ptr(umbrella), ptr(counts))
    total = lib.mw_triangulate(*args, None, 0, ptr(stats))
    tri = np.zeros((max(total, 1), 3), np.uint32)
    lib.mw_triangulate(*args, ptr(tri), total, ptr(stats))
    names = ("triangle_count", "vertices_meshed", "boundary_edges", "umbrella_overflows")
    return tri[:total], {k: int(v) for k, v in zip(names, stats)}, umbrella[:n], counts[:n]


class State:
    """One state's mesh and, per slot, what an update keeps: the umbrella (capped), the exact umbrella, the owned
    triangles, and the share of the stats (meshed, boundary edges of its directed edges, overflow)."""

    def __init__(self, rows, params=None):
        self.rows = np.ascontiguousarray(rows, np.float32)
        self.n = self.rows.shape[1]
        self.tri, self.stats, self.umbrella, self.count = walk(self.rows, params)
        _, _, wide, wide_count = walk(self.rows, params, WIDE)
        self.exact = [tuple(map(tuple, wide[i, :wide_count[i]].tolist())) for i in range(self.n)]
        self.overflow = wide_count > M.U
        tri = self.tri.astype(np.int64)
        self.owned = [[] for _ in range(self.n)]
        for t in tri.tolist():
            self.owned[t[0]].append(tuple(t))
        self.meshed = np.zeros(self.n, bool)
        self.meshed[np.unique(tri)] = True
        directed = np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [2, 0]]]) if len(tri) else np.zeros((0, 2), np.int64)
        present = {tuple(e) for e in directed.tolist()}
        self.boundary = np.zeros(self.n, np.int64)
        for a, b in directed.tolist():
            if (b, a) not in present:
                self.boundary[a] += 1

    def named(self, i):
        """Slots named in U(i), the umbrella the product keeps (empty on an overflow)."""
        return self.umbrella[i, :self.count[i]].ravel()

    def share(self, o):
        if o >= self.n:
            return ((), False, 0, False)
        return (tuple(self.owned[o]), bool(self.meshed[o]), int(self.boundary[o]), bool(self.overflow[o]))


def changed_set(old_rows, new_rows):
    """C: slots that are or were present whose snapshot bits differ; present slots beyond the old size."""
    n_old, n_new = old_rows.shape[1], new_rows.shape[1]
    n_max = max(n_old, n_new)
    out = np.zeros(n_max, bool)
    was = np.zeros(n_max, bool)
    now = np.zeros(n_max, bool)
    was[:n_old] = old_rows[7] > 0
    now[:n_new] = new_rows[7] > 0
    differ = np.ones(n_max, bool)
    k = min(n_old, n_new)
    rows = list(SNAPSHOT_ROWS)
    differ[:k] = (old_rows[rows, :k].view(np.uint32) != new_rows[rows, :k].view(np.uint32)).any(0)
    out = (was | now) & differ
    return out, was, now


def rebuild_set(old_rows, new_rows, params=None, strict=False):
    """A: C plus every present slot whose ball (rule 1's fp32 test) holds an old or new position of a slot of C.
    strict=True turns the test's <= into < (a deliberately wrong variant the tests must tell apart)."""
    p = params or L.MeshParams.defaults()
    c, was, now = changed_set(old_rows, new_rows)
    n = new_rows.shape[1]
    a = c[:n].copy()
    idx = np.flatnonzero(c)
    pts = [old_rows[3:6, i] for i in idx if was[i]] + [new_rows[3:6, i] for i in idx if now[i]]
    if not pts:
        return a, c
    pts = np.asarray(pts, np.float32)
    f = np.float32(p.neighbor_radius_factor)
    f2 = np.float32(f * f)
    r2 = new_rows[7]
    present = np.flatnonzero(r2 > 0)
    present = present[np.isfinite(new_rows[3:6, present]).all(0)]
    if not len(present):
        return a, c
    ball = (r2[present] * f2).astype(np.float32)
    reach = float(np.sqrt(ball.max())) * 1.001 + 1e-30
    tree = cKDTree(pts.astype(np.float64))
    near = tree.query_ball_point(new_rows[3:6, present].T.astype(np.float64), reach)
    with np.errstate(invalid="ignore", over="ignore"):
        for k, i in enumerate(present):
            if a[i] or not near[k]:
                continue
            q = pts[near[k]]
            d = q - new_rows[3:6, i][None, :]
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            a[i] = bool((d2 < ball[k]).any() if strict else (d2 <= ball[k]).any())
    return a, c


def recheck_set(old, a):
    """R: A plus every slot whose (kept) umbrella names a slot of A; a slot outside A has it unchanged."""
    n_max = max(old.n, len(a))
    r = np.zeros(n_max, bool)
    r[:len(a)] = a
    in_a = np.zeros(n_max + 1, bool)
    in_a[:len(a)] = a
    for o in range(min(old.n, len(a))):
        if not r[o] and in_a[old.named(o)].any():
            r[o] = True
    return r


def incremental(old, new, r):
    """The mesh an update assembles: old triangles and shares outside R, new ones inside it."""
    tri, stats = [], {"vertices_meshed": 0, "boundary_edges": 0, "umbrella_overflows": 0}
    for o in range(max(old.n, new.n)):
        owned, meshed, boundary, overflow = (new if r[o] else old).share(o)
        tri.extend(owned)
        stats["vertices_meshed"] += meshed
        stats["boundary_edges"] += boundary
        stats["umbrella_overflows"] += overflow
    stats["triangle_count"] = len(tri)
    return np.asarray(tri, np.uint32).reshape(-1, 3), stats


# ---- edit sequences ------------------------------------------------------------------------------------------

def _present(rows):
    return np.flatnonzero(rows[7] > 0)


def edit_sequence(rows, seed=0):
    """Cumulative edits of a state: [(label, rows)], each applied to the previous one."""
    rng = np.random.default_rng(seed)
    out = []
    cur = np.array(rows, np.float32, copy=True)

    def step(label, fn):
        nonlocal cur
        nxt = cur.copy()
        fn(nxt)
        out.append((label, nxt))
        cur = nxt

    live = _present(cur)
    if len(live) < 4:
        step("append", lambda r: None)
        return out
    pick = lambda: int(rng.choice(_present(cur)))
    i = pick()
    step("nudge_one_ulp", lambda r: r.__setitem__((3, i), np.nextafter(r[3, i], np.float32(np.inf))))
    j, k = pick(), pick()
    step("move_across", lambda r: r.__setitem__((slice(3, 6), j), r[3:6, k] + np.float32(1e-4)))
    g = pick()
    step("radius_grown", lambda r: r.__setitem__((7, g), r[7, g] * np.float32(2.5)))
    step("radius_shrunk", lambda r: r.__setitem__((7, g), r[7, g] * np.float32(0.1)))
    h = pick()
    step("normal_flipped", lambda r: r.__setitem__((slice(8, 11), h), -r[8:11, h]))
    v = pick()
    step("normal_invalid", lambda r: r.__setitem__((slice(8, 11), v), 0.0))
    m = pick()
    step("merged", lambda r: r.__setitem__((7, m), -1.0))

    def regularise(r):
        stamp = r.view(np.uint32)[24]
        lo = np.percentile(stamp, 40)
        sel = np.flatnonzero((stamp >= lo) & (stamp < lo + (stamp.max() - stamp.min()) * 0.1 + 1) & (r[7] > 0))
        r[3:6, sel] *= np.float32(1 + 1e-6)
    step("regularisation_window", regularise)

    src = rng.choice(_present(cur), 12)
    extra = cur[:, src].copy()
    extra[3:6] += np.float32(3e-4)
    cur = np.concatenate([cur, extra], 1)
    out.append(("append", cur))
    return out


def tie_sequence():
    """pixel_grid: a point moved one ulp off its cocircular quad, then back onto it."""
    rows = M.pixel_grid()
    side = 24
    i = side * (side // 2) + side // 2
    a = rows.copy()
    a[3, i] = np.nextafter(a[3, i], np.float32(np.inf))
    b = a.copy()
    b[3, i] = rows[3, i]
    return rows, [("tie_broken", a), ("tie_restored", b)]


def edge_sequence():
    """pixel_grid with a radius chosen so that the four diagonal neighbours lie exactly on the edge of each ball
    (d^2 == r^2 f^2 in fp32) and take part in its squares' triangles; then one slot leaves the sheet and comes back,
    which only the <= test of rule 1 notices for those diagonals."""
    spacing = np.float32(2.0 ** -7)
    rows = M.pixel_grid()
    rows[7] = (spacing * spacing) / np.float32(2.0)   # f = 2: the ball reaches exactly sqrt(2) spacings
    side = 24
    i = side * (side // 2) + side // 2
    a = rows.copy()
    a[5, i] = rows[5, i] + np.float32(1.0)
    b = a.copy()
    b[5, i] = rows[5, i]
    return rows, [("edge_away", a), ("edge_back", b)]
