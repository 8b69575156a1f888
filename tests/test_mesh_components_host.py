"""sm_mesh_components on the CPU: the plain-C restatement (tests/components_walk.c, sorted edges and a breadth-first
flood fill) checked against independent numpy / scipy code (scipy.sparse.csgraph.connected_components over the
shared-edge graph, numpy sums) on the hand-built meshes, every mesh_walk case and golden f7; pieces that touch at a
slot, a non-manifold edge, isolated triangles, ties in area, every threshold on both sides of its boundary, and the
header's rules. The GPU is held to the restatement bit for bit in tests/test_mesh_components_gpu.py.

Golden f7, meshed by the restated sm_triangulate: 21 217 triangles in 34 pieces; 11 pieces of fewer than 10
triangles (42 triangles), 19 of fewer than 50 (219 triangles); 0.942 m^2 in all.
"""
from pathlib import Path

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from surfelmeshing_b200._lib import ComponentParams
from tests import components_walk as CW
from tests import mesh_walk as M

CASES = CW.mesh_cases()


def ordered(f):
    """IEEE totalOrder of float32 values as uint32 keys."""
    b = np.asarray(f, np.float32).view(np.uint32)
    return np.where(b >> 31 == 1, ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def unordered(k):
    k = np.asarray(k, np.uint32)
    return np.where(k >> 31 == 1, k & np.uint32(0x7FFFFFFF), ~k).astype(np.uint32).view(np.float32)


def reference(rows, tri, p):
    """C2-C7 restated with scipy and numpy: (kept, labels, table fields, stats)."""
    tri = np.asarray(tri, np.int64).reshape(-1, 3)
    T = len(tri)
    if T == 0:
        return np.zeros((0, 3), np.int64), np.zeros(0, np.int64), None, dict.fromkeys(CW.STATS, 0)
    e = np.sort(np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [2, 0]]]), axis=1)
    owner = np.tile(np.arange(T), 3)
    order = np.lexsort((owner, e[:, 1], e[:, 0]))
    e, owner = e[order], owner[order]
    same = np.all(e[1:] == e[:-1], axis=1)              # consecutive entries of one undirected edge
    graph = coo_matrix((np.ones(int(same.sum())), (owner[:-1][same], owner[1:][same])), shape=(T, T))
    P, raw = connected_components(graph, directed=False)
    first = np.full(P, T)
    np.minimum.at(first, raw, np.arange(T))
    number = np.argsort(np.argsort(first))             # pieces numbered by their first triangle
    labels = number[raw]
    pos = rows[3:6].T.astype(np.float32)
    pd = pos.astype(np.float64)
    a, b, c = pd[tri[:, 0]], pd[tri[:, 1]], pd[tri[:, 2]]
    e1, e2 = b - a, c - a
    gx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    gy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    gz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    area = 0.5 * np.sqrt((gx * gx + gy * gy) + gz * gz)
    scaled = area * 2.0 ** 30
    q = np.where(np.isfinite(area), np.minimum(np.rint(scaled), 2.0 ** 36), 0)   # scaled = inf: the cap
    q = q.astype(np.uint64)
    counts = np.bincount(labels, minlength=P).astype(np.uint64)
    Q = np.zeros(P, np.uint64)
    np.add.at(Q, labels, q)
    lo = np.full((P, 3), 0xFFFFFFFF, np.uint32)
    hi = np.zeros((P, 3), np.uint32)
    for k in range(3):
        key = ordered(pos[tri[:, k]])
        np.minimum.at(lo, labels, key)
        np.maximum.at(hi, labels, key)
    rank = np.empty(P, np.int64)
    rank[sorted(range(P), key=lambda i: (-int(Q[i]), i))] = np.arange(P)
    units = np.rint(p.min_area * 2.0 ** 30)
    kept = (counts >= p.min_triangles) & (Q.astype(object) >= units if units >= 2.0 ** 63 else Q >= np.uint64(units))
    kept = np.asarray(kept, bool) & ((p.keep_largest == 0) | (rank < p.keep_largest))
    top = int(np.flatnonzero(rank == 0)[0])
    table = {"triangles": counts, "area": Q.astype(np.float64) * 2.0 ** -30, "lo": unordered(lo), "hi": unordered(hi),
             "first_triangle": np.sort(first).astype(np.uint32), "kept": kept.astype(np.int32)}
    stats = {"triangles_in": T, "triangles_out": int(kept[labels].sum()), "components": P,
             "components_kept": int(kept.sum()), "largest_triangles": int(counts[top]),
             "largest_area": float(Q[top]) * 2.0 ** -30}
    return tri[kept[labels]], labels, table, stats


def assert_matches_reference(rows, tri, p):
    out, labels, table, stats = CW.components(rows, tri, p)
    want_out, want_labels, want_table, want_stats = reference(rows, tri, p)
    assert stats == want_stats
    assert np.array_equal(out.astype(np.int64), want_out) and np.array_equal(labels, want_labels)
    if want_table is not None:
        for k, v in want_table.items():
            got = np.ascontiguousarray(table[k])
            assert np.array_equal(got.view(np.uint8), np.ascontiguousarray(v, got.dtype).view(np.uint8)), k
    return out, labels, table, stats


PARAMS = {"defaults": ComponentParams.defaults(), "all": ComponentParams.defaults(min_triangles=0),
          "largest_2": ComponentParams.defaults(min_triangles=0, keep_largest=2),
          "area": ComponentParams.defaults(min_triangles=1, min_area=1e-3)}


@pytest.mark.parametrize("params", sorted(PARAMS))
@pytest.mark.parametrize("name", sorted(CASES))
def test_walk_matches_scipy(name, params):
    rows, tri = CASES[name]
    assert_matches_reference(rows, tri, PARAMS[params])


@pytest.mark.parametrize("params", sorted(PARAMS))
def test_golden_f7(params):
    rows = M.golden_f7()
    tri, _, _ = M.triangulate(rows)
    out, labels, table, stats = assert_matches_reference(rows, tri, PARAMS[params])
    sizes = np.sort(table["triangles"])[::-1]
    assert len(tri) == 21217 and stats["components"] == 34
    assert sizes[:9].tolist() == [9112, 4057, 2792, 1891, 973, 745, 509, 289, 261]
    small = sizes < 10
    assert small.sum() == 11 and sizes[small].sum() == 42 and abs(table["area"][table["triangles"] < 10].sum() - 1.2e-3) < 1e-4
    assert (sizes < 50).sum() == 19 and sizes[sizes < 50].sum() == 219
    assert abs(table["area"].sum() - 0.942) < 1e-3
    if params == "defaults":
        assert stats["components_kept"] == 23 and stats["triangles_out"] == 21217 - 42


def test_pieces_touching_at_one_slot_stay_two():
    rows, tri = CASES["touching_planes"]
    _, labels, table, stats = CW.components(rows, tri, ComponentParams.defaults(min_triangles=0))
    assert stats["components"] == 2 and labels.tolist() == [0] * 6 + [1] * 6
    assert table["first_triangle"].tolist() == [0, 6]


def test_non_manifold_edge_is_one_piece():
    rows, tri = CASES["fin"]
    out, labels, table, stats = CW.components(rows, tri, ComponentParams.defaults(min_triangles=0))
    assert stats["components"] == 1 and labels.tolist() == [0, 0, 0, 0] and len(out) == 4
    # bounds: every corner's smooth position
    pos = rows[3:6].T
    assert np.array_equal(table["lo"][0], pos.min(0)) and np.array_equal(table["hi"][0], pos.max(0))


def test_isolated_triangles_and_the_rank_tie_break():
    rows, tri = CASES["islands"]
    p = ComponentParams.defaults(min_triangles=0)
    _, labels, table, stats = CW.components(rows, tri, p)
    assert table["triangles"].tolist() == [1, 8, 1, 12, 8]
    assert table["first_triangle"].tolist() == [0, 1, 9, 10, 22]
    assert table["area"][1] == table["area"][4]                           # a tie in Q: the smaller number ranks first
    assert stats["largest_triangles"] == 12 and stats["largest_area"] == table["area"][3]
    for k, kept in ((1, [3]), (2, [1, 3]), (3, [1, 3, 4]), (4, [0, 1, 3, 4]), (5, [0, 1, 2, 3, 4]), (9, [0, 1, 2, 3, 4])):
        out, _, table, stats = CW.components(rows, tri, ComponentParams.defaults(min_triangles=0, keep_largest=k))
        assert np.flatnonzero(table["kept"]).tolist() == kept, k
        assert np.array_equal(out, np.asarray(tri)[np.isin(labels, kept)])


def test_thresholds_on_both_sides_of_their_boundary():
    rows, tri = CASES["islands"]
    _, _, table, _ = CW.components(rows, tri, ComponentParams.defaults(min_triangles=0))
    Q = np.rint(table["area"] * 2.0 ** 30).astype(np.int64)
    assert np.array_equal(Q.astype(np.float64) * 2.0 ** -30, table["area"])

    def kept(**kw):
        return np.flatnonzero(CW.components(rows, tri, ComponentParams.defaults(**kw))[2]["kept"]).tolist()
    assert kept(min_triangles=8) == [1, 3, 4] and kept(min_triangles=9) == [3]
    assert kept(min_triangles=12) == [3] and kept(min_triangles=13) == []
    assert kept(min_triangles=0) == kept(min_triangles=1) == [0, 1, 2, 3, 4]
    q8 = int(Q[1])
    # min_area exactly at the 8-triangle pieces' area units, one unit above, and half a unit either side (ties to even)
    assert kept(min_triangles=0, min_area=q8 * 2.0 ** -30) == [1, 3, 4]
    assert kept(min_triangles=0, min_area=(q8 + 1) * 2.0 ** -30) == [3]
    half_up = [1, 3, 4] if (q8 % 2 == 0) else [3]
    assert kept(min_triangles=0, min_area=(q8 + 0.5) * 2.0 ** -30) == half_up
    assert kept(min_triangles=0, min_area=(q8 - 0.5) * 2.0 ** -30) == [1, 3, 4]
    assert kept(min_triangles=0, min_area=1e300) == []


def test_area_units_rounding_and_cap():
    """q_t = rint(a_t * 2^30), ties to even, capped at 2^36; a triangle of area 2^-31 m^2 is half a unit."""
    s = 2.0 ** -15   # legs of 2^-15 m: area 2^-31
    pos = [[0, 0, 1], [s, 0, 1], [0, s, 1], [0, 0, 2], [3 * s, 0, 2], [0, s, 2], [0, 0, 3], [3e5, 0, 3], [0, 3e5, 3]]
    rows = M.make_rows(pos, (0, 0, 1), 1e-4)
    tri = [(0, 1, 2), (3, 4, 5), (6, 7, 8)]
    _, _, table, _ = CW.components(rows, tri, ComponentParams.defaults(min_triangles=0))
    assert table["area"].tolist() == [0.0, 2.0 * 2.0 ** -30, 2.0 ** 6]   # 0.5 -> 0, 1.5 -> 2, 4.5e10 m^2 -> 2^36 units


def test_invalid_inputs_are_refused():
    rows, tri = CASES["islands"]
    n = rows.shape[1]
    with pytest.raises(CW.InvalidMesh, match="bad corner"):
        CW.components(rows, np.concatenate([tri, [[0, 1, n]]]))
    with pytest.raises(CW.InvalidMesh, match="repeated corner"):
        CW.components(rows, np.concatenate([tri, [[0, 0, 1]]]))
    for padding in ([[0, -1, -1]], [[-1, -1, -1]]):   # -1 corners: bad (and repeated)
        with pytest.raises(CW.InvalidMesh, match="bad corner"):
            CW.components(rows, np.concatenate([tri, padding]))
    merged = rows.copy()
    merged[7, 5] = -merged[7, 5]
    with pytest.raises(CW.InvalidMesh, match="bad corner"):
        CW.components(merged, tri)
    out, labels, table, stats = CW.components(rows, np.zeros((0, 3)))
    assert len(out) == len(labels) == len(table) == 0 and stats == dict.fromkeys(CW.STATS, 0)


def test_header_declares_the_call():
    h = (Path(__file__).resolve().parents[1] / "include" / "surfel_b200.h").read_text()
    assert "int sm_mesh_components(" in h and "} sm_mesh_component;" in h
    for rule in ("C1. Input.", "C2. Adjacency.", "C3. Numbering.", "C4. Area.", "C5. Bounds.", "C6. Keep.", "C7. Output."):
        assert rule in h
