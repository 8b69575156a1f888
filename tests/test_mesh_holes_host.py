"""sm_mesh_fill_holes on the CPU: the plain-C restatement (tests/hole_walk.c) on hand-built triangle lists over
mesh_walk clouds, on every mesh_walk case and on golden f7; the invariants of mesh and fill together, the reference
mesher's area where it is built, and the ABI. The GPU is held to the restatement bit for bit in
tests/test_mesh_holes_gpu.py.

Observed with the restatement (default parameters but K) when these tests were written:
  sphere (2000 slots)        4 quad holes, 16 boundary edges: 8 triangles close it (V - E + F = 2)
  sheet                      14 loops (7 quads, 4 five-edge and 3 six-edge holes), all filled
  golden f7, K = 4 / 8 / 16  55 / 62 / 78 loops, 52 / 53 / 59 filled, 78 / 82 / 154 triangles
"""
from pathlib import Path

import numpy as np
import pytest

from surfelmeshing_b200._lib import HoleParams
from tests import hole_walk as HW
from tests import mesh_walk as M

SIDE = 8


def fill(rows, tri, K=8, normals=90.0, angle=180.0):
    return HW.fill_holes(rows, tri, HoleParams(K, normals, angle))


def test_one_missing_triangle_comes_back():
    rows, tri = HW.grid_mesh(SIDE)
    for i, j, r in ((2, 2, 0), (3, 4, 1), (5, 1, 0)):   # interior squares: (i, j) -> triangles 2 (i (side - 1) + j) + r
        drop = 2 * (i * (SIDE - 1) + j) + r
        f, s = fill(rows, np.delete(tri, drop, 0))
        assert f.tolist() == [tri[drop].tolist()]
        assert s["loops_filled"] == 1 and s["boundary_edges_after"] == s["boundary_edges"] - 3


def test_ring_of_a_removed_slot_is_filled():
    rows, tri = HW.grid_mesh(SIDE)
    centre = 3 * SIDE + 4
    mesh = HW.without(tri, [centre])
    f, s = fill(rows, mesh)
    assert s["loops_found"] == s["loops_filled"] == 1 and len(f) == 4
    V, E, F, B, loops = HW.check_union(rows, mesh, f)
    assert loops == 1 and B == 4 * (SIDE - 1)   # only the outer boundary remains
    full = (SIDE - 1) ** 2 * 2.0 ** -14
    assert abs(M.area(rows, np.concatenate([mesh, f]).astype(np.int64)) / full - 1) < 1e-6


def test_two_square_holes_sharing_a_vertex_are_both_filled():
    # squares (2, 2) and (3, 3) touch at slot (3, 3): two hole edges leave it, and rule H2 must pair each incoming
    # edge with the outgoing edge of its own square (clockwise from the incoming one)
    rows, tri = HW.grid_mesh(SIDE)
    mesh = HW.without_triangles(tri, np.concatenate([HW.square_hole(SIDE, 2, 2), HW.square_hole(SIDE, 3, 3)]))
    f, s = fill(rows, mesh)
    assert s["loops_found"] == s["loops_filled"] == 2 and len(f) == 4
    assert HW.check_union(rows, mesh, f)[3] == 4 * (SIDE - 1)
    pinch = 3 * SIDE + 3
    assert (f == pinch).any(1).sum() == 2 and np.isin(f, HW.square_hole(SIDE, 2, 2)).all(1).sum() == 2


def test_hole_whose_diagonals_exist_elsewhere_is_rejected():
    # Both diagonals of a square hole are made input edges by two closed two-triangle pillows over extra slots.
    rows, tri = HW.grid_mesh(SIDE)
    extra = M.make_rows([[0.5, 0.5, 3.0], [0.6, 0.4, 3.0]], (0, 0, 1), 1e-4)
    rows = np.concatenate([rows, extra], 1)
    z, w = SIDE * SIDE, SIDE * SIDE + 1
    sq = HW.square_hole(SIDE, 2, 2)
    a, b, c, d = 2 * SIDE + 2, 3 * SIDE + 2, 3 * SIDE + 3, 2 * SIDE + 3
    mesh = HW.without_triangles(tri, sq)
    f, s = fill(rows, mesh)
    assert s["loops_filled"] == 1
    pillows = HW.canonical([(a, c, z), (c, a, z), (b, d, w), (d, b, w)])
    f, s = fill(rows, np.concatenate([mesh, pillows]))
    assert s["loops_found"] == 1 and s["loops_rejected"] == 1 and len(f) == 0
    assert s["boundary_edges_after"] == s["boundary_edges"] == 4 * (SIDE - 1) + 4


def test_nothing_is_filled_across_the_normal_gate():
    rows = M.crossing_planes(30)
    tri, _, _ = M.triangulate(rows)
    half = rows.shape[1] // 2
    for K in (4, 8, 16):
        f, _ = fill(rows, tri, K, normals=20.0)
        side = f.astype(np.int64) >= half
        assert (side.all(1) | (~side).all(1)).all(), "a fill triangle joins the two planes"


def test_normal_gate_decides():
    rows, tri = HW.tilted_corner_case(45.0)   # one corner of a square hole tilted by 45 degrees
    for gate in (90.0, 50.0):
        f, s = fill(rows, tri, normals=gate)
        assert s["loops_filled"] == 1 and len(f) == 2
    for gate in (40.0, 30.0):
        f, s = fill(rows, tri, normals=gate)
        assert s["loops_rejected"] == 1 and len(f) == 0


def test_triangle_angle_decides():
    rows, tri = HW.angle_case()
    f, _ = fill(rows, tri, 4, angle=180.0)
    assert f.tolist() == [[0, 2, 3], [0, 1, 2]]   # the smaller split has an angle above 120 degrees
    f, _ = fill(rows, tri, 4, angle=120.0)
    assert f.tolist() == [[0, 1, 3], [1, 2, 3]]
    f, s = fill(rows, tri, 4, angle=60.0)
    assert len(f) == 0 and s["loops_rejected"] == 1


def test_two_loops_proposing_one_diagonal_are_both_dropped():
    rows, a, b, both = HW.conflict_case()
    fa, sa = fill(rows, a, normals=180.0)
    fb, sb = fill(rows, b, normals=180.0)
    assert sa["loops_filled"] == 1 and len(fa) == 4 and sb["loops_filled"] == 1 and len(fb) == 2
    diagonal = {0, 3}
    assert any(diagonal <= set(t) for t in fa.tolist()) and any(diagonal <= set(t) for t in fb.tolist())
    f, s = fill(rows, both, normals=180.0)
    assert s["loops_found"] == 2 and s["loops_conflicting"] == 2 and len(f) == 0
    assert s["boundary_edges_after"] == s["boundary_edges"] == 10
    f, s = fill(rows, both, normals=90.0)   # the gate rejects both before they can conflict
    assert s["loops_rejected"] == 2 and s["loops_conflicting"] == 0


def test_outer_boundary_is_left_open_below_its_length():
    rows, tri = HW.grid_mesh(3)   # outer boundary: 8 edges, no other hole
    for K in (3, 4, 7):
        f, s = fill(rows, tri, K)
        assert s["loops_found"] == 0 and len(f) == 0 and s["boundary_edges_after"] == 8
    f, s = fill(rows, tri, 8)   # a loop of 8, oriented against the normals: every triangle fails H4
    assert s["loops_found"] == 1 and s["loops_rejected"] == 1 and len(f) == 0


def test_sphere_is_closed():
    rows = M.sphere()
    tri, _, _ = M.triangulate(rows)
    f, s = fill(rows, tri, 4)
    assert s["boundary_edges"] == 16 and s["loops_filled"] == 4
    V, E, F, B, _ = HW.check_union(rows, tri, f)
    assert V - E + F == 2 and B == 0 and s["boundary_edges_after"] == 0


def test_sheet_holes_are_filled():
    rows = M.meshing_cloud("sheet")
    tri, _, _ = M.triangulate(rows)
    f, s = fill(rows, tri, 6)
    assert s["loops_found"] == s["loops_filled"] == 14
    assert len(f) == 7 * 2 + 4 * 3 + 3 * 4


@pytest.mark.parametrize("K", [3, 4, 8, 16])
@pytest.mark.parametrize("name", sorted(M.CASES) + ["golden_f7"])
def test_invariants_of_mesh_and_fill(name, K):
    rows = M.golden_f7() if name == "golden_f7" else M.CASES[name]()
    tri, _, _ = M.triangulate(rows)
    f, s = fill(rows, tri, K)
    _, _, _, B, _ = HW.check_union(rows, tri, f)
    assert s["boundary_edges"] == M.topology(tri)[3]
    assert s["boundary_edges_after"] == B
    assert s["loops_filled"] + s["loops_rejected"] + s["loops_conflicting"] == s["loops_found"]
    assert s["triangles_added"] == len(f)
    # every filled loop of k edges adds k - 2 triangles and closes k boundary edges
    assert s["boundary_edges"] - s["boundary_edges_after"] == len(f) + 2 * s["loops_filled"]


def test_invalid_inputs_are_refused():
    rows, tri = HW.grid_mesh(4)
    n = rows.shape[1]
    with pytest.raises(HW.InvalidMesh, match="bad corner"):
        fill(rows, np.concatenate([tri, [[0, 1, n]]]))
    merged = rows.copy()
    merged[7, 5] = -merged[7, 5]
    with pytest.raises(HW.InvalidMesh, match="bad corner"):
        fill(merged, tri)
    with pytest.raises(HW.InvalidMesh, match="repeated corner"):
        fill(rows, np.concatenate([tri, [[0, 0, 1]]]))
    with pytest.raises(HW.InvalidMesh, match="duplicate edge"):
        fill(rows, np.concatenate([tri, tri[:1]]))


def test_area_moves_toward_the_reference_mesher():
    from oracle import meshing_ref
    if not meshing_ref.available():
        pytest.skip("oracle/_ref/libmeshing_ref.so not built")
    rows = M.golden_f7()
    tri, _, _ = M.triangulate(rows)
    ref = meshing_ref.SurfelMeshing()
    ref.integrate(1, *[rows[k] for k in (3, 4, 5, 7, 8, 9, 10)], rows[18].view(np.uint32))
    ref.check_remeshing()
    ref.triangulate()
    ref_area = M.area(rows, ref.triangles())
    ref.close()
    before = M.area(rows, tri) / ref_area
    last = before
    for K in (4, 8, 16):
        f, _ = fill(rows, tri, K)
        ratio = M.area(rows, np.concatenate([tri, f]).astype(np.int64)) / ref_area
        print(f"K = {K}: area {ratio:.4f} of the reference's (mesh alone {before:.4f})")
        assert last <= ratio <= 1.02
        last = ratio
    assert last > before


def test_header_declares_the_call():
    h = (Path(__file__).resolve().parents[1] / "include" / "surfel_b200.h").read_text()
    assert "int sm_mesh_fill_holes(" in h and "void sm_default_hole_params(sm_hole_params* p);" in h
