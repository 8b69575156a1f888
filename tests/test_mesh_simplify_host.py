"""sm_mesh_simplify on the CPU: the plain-C restatement (tests/simplify_walk.c) on hand-built meshes, on the restated
meshes of mesh_walk clouds and on golden f7 with its fill; what a simplified mesh keeps (boundary, Euler
characteristic, area of a plane, manifoldness), the rules that stop a collapse, the budget round, the OBJ export of
the referenced slots. The walk applies every round in both orders and raises if they differ, so every
case here also checks S4. The GPU is held to the restatement bit for bit in tests/test_mesh_simplify_gpu.py.

Observed with the restatement when these tests were written (default parameters unless stated):
  pixel_grid, max_cost 0       1058 -> 90 triangles (only the 92 boundary slots remain)
  jittered_plane, max_cost 0   1713 -> 423 triangles in the 64 rounds of the default (x 4.05)
  octahedron, no bounds        8 -> 4 triangles in two rounds, then nothing is valid
"""
import math

import numpy as np
import pytest

from surfelmeshing_b200 import _lib, mesh_io
from surfelmeshing_b200._lib import SimplifyParams
from tests import hole_walk as HW
from tests import mesh_walk as M
from tests import simplify_walk as SW


def euler(tri):
    V, E, F, _, _ = M.topology(tri)
    return V - E + F


def check_kept(rows, tri, out, stats):
    """The invariants of S8 and the stats every call must satisfy."""
    M.check_invariants(rows, out)
    before, after = M.topology(tri), M.topology(out)
    assert after[3] == before[3], "boundary edges"
    assert euler(out) == euler(tri)
    assert stats["triangles_in"] == len(tri) and stats["triangles_out"] == len(out)
    assert stats["vertices_in"] == before[0] and stats["vertices_out"] == after[0]
    assert stats["boundary_edges"] == before[3]
    assert len(tri) - len(out) == 2 * stats["collapses"]
    assert before[0] - after[0] == stats["collapses"]
    # the boundary edges themselves, so the boundary loops too (topology() counts loops through pinch vertices by
    # the order of its dictionary, so its count is compared only where a case has none)
    def boundary(t):
        t = np.asarray(t, np.int64).reshape(-1, 3)
        e = {tuple(x) for x in np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]).tolist()}
        return {x for x in e if (x[1], x[0]) not in e}
    assert boundary(out) == boundary(tri)


@pytest.mark.parametrize("name", ["pixel_grid", "jittered_plane"])
def test_plane_keeps_boundary_and_area(name):
    rows = M.CASES[name]()
    tri = SW.meshed(rows)
    out, s = SW.simplify(rows, tri, SimplifyParams.defaults(max_cost=0.0))
    check_kept(rows, tri, out, s)
    assert M.topology(out)[3:] == M.topology(tri)[3:] == (M.topology(tri)[3], 1)
    assert abs(M.area(rows, out) / M.area(rows, tri) - 1) <= 1e-12
    print(f"{name}: {len(tri)} -> {len(out)} triangles in {s['rounds']} rounds")
    assert 4 * len(out) <= len(tri)


def test_octahedron_ends_as_a_tetrahedron():
    rows, tri = SW.octahedron()
    out, s, log = SW.simplify(rows, tri, SW.unbounded(), log=True)
    check_kept(rows, tri, out, s)
    assert len(out) == 4 and s["vertices_out"] == 4 and s["stop_reason"] == _lib.SIMPLIFY_STOP_CONVERGED
    assert log["rounds"] == [(1, 1), (1, 1)]   # every closed neighbourhood of an octahedron overlaps every other
    # a tetrahedron's collapses pass the link condition; with normals pointing outwards, the moved triangle faces
    # inwards and fails rule (c)'s orientation test (test_repeated_triangle_decides has normals where it does not)
    out2, s2 = SW.simplify(rows, out, SW.unbounded())
    assert np.array_equal(out2, out) and s2["collapses"] == 0


def test_crease_is_kept():
    rows = M.crossing_planes(90)
    tri = SW.meshed(rows)
    out, s = SW.simplify(rows, tri, SimplifyParams.defaults(max_cost=1e-12))
    check_kept(rows, tri, out, s)
    assert s["collapses"] > 0
    # slots of the first plane are < half, of the second >= half; y == 0 is the crease, shared by both planes
    half = rows.shape[1] // 2
    on_crease = np.abs(rows[4] - rows[4, :half].mean()) < 1e-6
    first = (np.arange(rows.shape[1]) < half) & ~on_crease
    second = (np.arange(rows.shape[1]) >= half) & ~on_crease
    assert not (first[out].any(1) & second[out].any(1)).any(), "a triangle joins the two planes off the crease"


def test_sphere_stays_closed_at_a_quarter():
    rows = M.sphere()
    tri = SW.meshed(rows)
    target = len(tri) // 4
    out, s = SW.simplify(rows, tri, SW.unbounded(target_triangles=target, max_angle_between_normals_deg=90.0,
                                                 max_triangle_angle_deg=170.0))
    check_kept(rows, tri, out, s)
    V, E, F, B, _ = M.topology(out)
    assert B == 0 and V - E + F == 2
    assert len(out) in (target, target - 1) and s["stop_reason"] == _lib.SIMPLIFY_STOP_TARGET


def quadric_costs(rows, tri, u):
    """{v: cost of u -> v} in float64 (S1's quadrics, not its rounding), over u's neighbours."""
    p = rows[3:6].T.astype(np.float64)
    tri = np.asarray(tri, np.int64)
    Q = np.zeros((rows.shape[1], 4, 4))
    for a, b, c in tri:
        g = np.cross(p[b] - p[a], p[c] - p[a])
        m = g / np.linalg.norm(g)
        plane = np.append(m, -m @ p[a])
        for i in (a, b, c):
            Q[i] += np.outer(plane, plane)
    ring = {int(x) for t in tri if u in t for x in t} - {u}
    return {v: float(np.append(p[v], 1) @ (Q[u] + Q[v]) @ np.append(p[v], 1)) for v in ring}


def test_neck_stays_closed():
    rows, tri = SW.neck()
    neck = {4, 5, 6}
    # the cheapest collapse of a neck slot is onto another neck slot, which would pinch the surface; here rule (c)'s
    # orientation test already refuses it (test_link_condition_decides has a collapse only the link condition stops)
    for u in neck:
        costs = quadric_costs(rows, tri, u)
        assert min(costs, key=costs.get) in neck
    out, s = SW.simplify(rows, tri, SW.unbounded())
    check_kept(rows, tri, out, s)
    V, E, F, B, _ = M.topology(out)
    assert B == 0 and V - E + F == 2


def moved_triangles_face_their_normals(rows, moved):
    p = rows[3:6].T.astype(np.float64)
    n = rows[8:11].T.astype(np.float64)
    for x, y, z in moved:
        g = np.cross(p[y] - p[x], p[z] - p[x])
        if not all(g @ n[c] > 0 for c in (x, y, z)):
            return False
    return True


def directed_edges_unique(tri):
    tri = np.asarray(tri, np.int64).reshape(-1, 3)
    edges = np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [2, 0]]])
    return len(np.unique(edges, axis=0)) == len(edges)


def test_link_condition_decides():
    rows, tri = SW.link_case()
    ring = {1, 2, 3, 4}
    N1 = {int(x) for t in tri if 1 in t for x in t} - {1}
    # 0 -> 1 passes every rule but (a): the ring (1, 2, 3, 4) has o1 = 4 and o2 = 2, but N(0) and N(1) share 3 too
    assert ring & N1 == {2, 3, 4}
    assert len(ring) + len(N1) - 4 <= _lib.MESH_MAX_VALENCE
    assert moved_triangles_face_their_normals(rows, [(1, 2, 3), (1, 3, 4)])
    assert not {frozenset(t) for t in tri.tolist()} & {frozenset((1, 2, 3)), frozenset((1, 3, 4))}
    assert (rows[5, :5] == 0).all()   # the fan and slot 1 lie on z = 0: the cost is 0
    # so slot 0 goes to 2 instead, the next smallest of its cost-0 neighbours, and the surface stays a sphere
    for p in (SW.unbounded(), SimplifyParams.defaults(max_cost=0.0)):
        out, s = SW.simplify(rows, tri, p)
        assert s["collapses"] == 1 and 0 not in out
        assert out.tolist() == [[1, 2, 4], [1, 4, 5], [1, 5, 3], [1, 3, 6], [1, 6, 2], [2, 3, 4], [2, 6, 3], [3, 5, 4]]
        assert directed_edges_unique(out) and euler(out) == 2 and M.topology(out)[3] == 0


def test_repeated_triangle_decides():
    rows, tri = SW.repeat_case()
    # collapsing the apex 0 onto a base corner v moves one triangle: the base with the other winding; the link
    # condition holds (degree 3), and every normal is +z, so the moved triangle faces all its corner normals
    for v, moved in ((1, (1, 2, 3)), (2, (2, 3, 1)), (3, (3, 1, 2))):
        assert moved_triangles_face_their_normals(rows, [moved])
        assert frozenset(moved) in {frozenset(t) for t in tri.tolist()}
    out, s = SW.simplify(rows, tri, SW.unbounded())
    assert np.array_equal(out, tri) and s["collapses"] == 0 and s["stop_reason"] == _lib.SIMPLIFY_STOP_CONVERGED


def test_budget_round_applies_the_smallest_keys():
    rows = M.CASES["jittered_plane"]()
    tri = SW.meshed(rows)
    target = len(tri) - 131   # inside a round: the first rounds select more than 66 collapses
    out, s, log = SW.simplify(rows, tri, SimplifyParams.defaults(max_cost=0.0, target_triangles=target), log=True)
    check_kept(rows, tri, out, s)
    R = s["rounds"]
    assert s["stop_reason"] == _lib.SIMPLIFY_STOP_TARGET and R >= 1
    before, _ = SW.simplify(rows, tri, SimplifyParams.defaults(max_cost=0.0, max_rounds=R - 1))
    full, _, full_log = SW.simplify(rows, tri, SimplifyParams.defaults(max_cost=0.0, max_rounds=R), log=True)
    T = len(before)
    applied = math.ceil((T - target) / 2)
    selected, last = log["rounds"][-1]
    assert last == applied and selected > applied and full_log["rounds"][-1] == (selected, selected)
    assert len(out) == T - 2 * applied and len(out) in (target, target - 1)
    keys = full_log["last_selected"]
    assert len(keys) == selected and (np.diff(keys.astype(np.float64)) > 0).all()
    removed = set(np.unique(before).tolist()) - set(np.unique(out).tolist())
    assert removed == {int(k) & 0xFFFFFFFF for k in keys[:applied]}


def test_valence_cap_holds_the_hub():
    rows, tri = SW.hub(40)
    out, s, log = SW.simplify(rows, tri, SW.unbounded(max_cost=0.0, max_rounds=8), log=True)
    check_kept(rows, tri, out, s)
    # every cost is 0, so each ring slot would pick the hub (slot 0, the smallest) were its valence in range; one
    # ring slot per round wins (all their closed neighbourhoods hold the hub), so the hub keeps 32 spokes or more
    assert log["rounds"] == [(1, 1)] * 8
    spokes = {int(x) for t in out if 0 in t for x in t} - {0}
    assert 0 in out and spokes <= set(range(1, 41)) and len(spokes) == 32


def test_max_rounds_zero_checks_and_reorders():
    rows, tri = HW.grid_mesh(6)
    shuffled = tri[np.random.default_rng(0).permutation(len(tri))]
    shuffled = np.roll(shuffled, 1, axis=1)   # every triangle starts at another corner
    out, s = SW.simplify(rows, shuffled, SimplifyParams.defaults(max_rounds=0))
    assert s["stop_reason"] == _lib.SIMPLIFY_STOP_MAX_ROUNDS and s["collapses"] == 0
    canon = HW.canonical(shuffled)
    assert np.array_equal(out, canon[np.lexsort((np.arange(len(canon)), canon[:, 0]))])
    M.check_invariants(rows, out)


@pytest.mark.parametrize("name", sorted(SW.mesh_cases()))
def test_invariants_on_every_case(name):
    rows, tri = SW.mesh_cases()[name]
    for p in (SimplifyParams.defaults(), SimplifyParams.defaults(max_cost=0.0),
              SW.unbounded(target_triangles=max(len(tri) // 4, 1), max_rounds=64)):
        out, s = SW.simplify(rows, tri, p)
        check_kept(rows, tri, out, s)


@pytest.mark.parametrize("fraction", [0.5, 0.25, 0.1])
def test_golden_f7_with_fill(fraction):
    rows = M.golden_f7()
    tri = SW.meshed(rows)
    target = int(len(tri) * fraction)
    for p in (SimplifyParams.defaults(target_triangles=target), SW.unbounded(target_triangles=target, max_rounds=64,
                                                                             max_angle_between_normals_deg=90.0,
                                                                             max_triangle_angle_deg=170.0)):
        out, s = SW.simplify(rows, tri, p)
        check_kept(rows, tri, out, s)
        print(f"golden f7, target {fraction:.0%} of {len(tri)}, max_cost {p.max_cost:g}: {len(out)} triangles, "
              f"{s['rounds']} rounds")


def test_invalid_inputs_are_refused():
    rows, tri = HW.grid_mesh(4)
    n = rows.shape[1]
    with pytest.raises(SW.InvalidMesh, match="bad corner"):
        SW.simplify(rows, np.concatenate([tri, [[0, 1, n]]]))
    with pytest.raises(SW.InvalidMesh, match="repeated corner"):
        SW.simplify(rows, np.concatenate([tri, [[0, 0, 1]]]))
    with pytest.raises(SW.InvalidMesh, match="duplicate edge"):
        SW.simplify(rows, np.concatenate([tri, tri[:1]]))
    out, s = SW.simplify(rows, np.zeros((0, 3), np.uint32))
    assert len(out) == 0 and s["stop_reason"] == _lib.SIMPLIFY_STOP_CONVERGED


def test_write_obj_referenced_only(tmp_path):
    positions = np.array([[0, 0, 0], [1, 0, 0], [np.nan, 0, 0], [0, 1, 0], [5, 5, 5], [1, 1, 0]], np.float32)
    colors = np.arange(18, dtype=np.uint8).reshape(6, 3)
    tri = np.array([[0, 1, 5], [0, 5, 3]])
    assert mesh_io.write_obj(tmp_path / "all.obj", positions, colors, tri) == (5, 2)
    assert mesh_io.write_obj(tmp_path / "used.obj", positions, colors, tri, referenced_only=True) == (4, 2)
    v_all, _, f_all = mesh_io.read_obj(tmp_path / "all.obj")
    v, c, f = mesh_io.read_obj(tmp_path / "used.obj")
    assert np.allclose(v, positions[[0, 1, 3, 5]]) and np.allclose(c * 255, colors[[0, 1, 3, 5]])
    assert np.allclose(v[f], v_all[f_all])   # the same faces, over fewer vertices
    assert f.tolist() == [[0, 1, 3], [0, 3, 2]]
    with pytest.raises(ValueError):
        mesh_io.write_obj(tmp_path / "bad.obj", positions, colors, [[0, 1, 2]], referenced_only=True)
