"""sm_triangulate on the CPU: the plain-C restatement (tests/mesh_walk.c) on hand-built clouds and the golden f7
state, the mesh invariants the rules guarantee, geometry bounds, the OBJ / PLY writers and the struct layouts.
The GPU kernels are compared with the restatement bit for bit in tests/test_mesh_gpu.py.

Observed with the restatement (default parameters) when these bounds were set:
  jittered plane (900 slots)  1713 triangles, chi = 1, one boundary loop, area 0.08492 vs 0.0841 for the square
  pixel grid (24 x 24)        1058 triangles = every unit square split in two, chi = 1, one loop
  sphere (2000 slots)         3988 of 3996 triangles, 16 boundary edges (4 small holes where the tangent planes of
                              nearly cocircular neighbours disagree about a diagonal)
  golden f7 (11 899 slots)    21 217 triangles, 2 445 boundary edges = 7.4 % of 33 048 edges, 11 794 slots meshed
"""
import ctypes as C

import numpy as np
import pytest

from surfelmeshing_b200 import _lib, mesh_io
from tests import mesh_walk as M


@pytest.mark.parametrize("name", sorted(M.CASES) + ["golden_f7"])
def test_invariants_hold_on_every_case(name):
    rows = M.golden_f7() if name == "golden_f7" else M.CASES[name]()
    tri, stats, _ = M.triangulate(rows)
    M.check_invariants(rows, tri)
    V, E, F, B, _ = M.topology(tri)
    assert stats["triangle_count"] == F
    assert stats["boundary_edges"] == B
    assert stats["vertices_meshed"] == V
    assert stats["umbrella_overflows"] == 0


def test_jittered_plane_is_one_disk_of_the_sampled_area():
    rows = M.jittered_plane()
    tri, _, _ = M.triangulate(rows)
    V, E, F, B, loops = M.topology(tri)
    assert V == rows.shape[1]
    assert V - E + F == 1 and loops == 1
    assert abs(M.area(rows, tri) / (29 * 0.01) ** 2 - 1) < 0.03


def test_pixel_grid_splits_every_square():
    rows = M.pixel_grid()
    tri, _, _ = M.triangulate(rows)
    V, E, F, B, loops = M.topology(tri)
    assert F == 2 * 23 * 23 and V - E + F == 1 and loops == 1 and B == 4 * 23


def test_sphere_is_nearly_closed():
    rows = M.sphere()
    tri, stats, _ = M.triangulate(rows)
    V, E, F, B, _ = M.topology(tri)
    assert V == rows.shape[1]
    assert F >= 0.995 * (2 * V - 4)
    assert B <= 0.005 * E
    assert abs(M.area(rows, tri) / (4 * np.pi * 0.25) - 1) < 0.02


@pytest.mark.parametrize("degrees", [90, 30])
def test_crossing_planes_do_not_mesh_across_the_gate(degrees):
    rows = M.crossing_planes(degrees)
    tri, _, _ = M.triangulate(rows)
    half = rows.shape[1] // 2
    side = np.asarray(tri, np.int64) >= half
    assert (side.all(1) | (~side).all(1)).all(), "a triangle joins the two planes"


def test_merged_and_gated_slots_are_not_corners():
    rows = M.with_merged()
    tri, _, _ = M.triangulate(rows)
    assert not np.isin(np.flatnonzero(rows[7] <= 0), tri).any()
    rows = M.with_flipped_normals()
    tri, _, _ = M.triangulate(rows)
    flipped = np.flatnonzero(rows[10] < 0)
    t = np.asarray(tri, np.int64)
    mixed = np.isin(t, flipped).any(1) & ~np.isin(t, flipped).all(1)
    assert not mixed.any(), "a triangle joins slots whose normals are 180 degrees apart"


def test_duplicate_positions_mesh_once():
    rows = M.with_duplicates()
    tri, _, _ = M.triangulate(rows)
    p = rows[3:6].T
    t = np.asarray(tri, np.int64)
    # no triangle has two corners at one position
    for a, b in ((0, 1), (1, 2), (0, 2)):
        assert not (p[t[:, a]] == p[t[:, b]]).all(1).any()


def test_golden_cloud_boundary_fraction():
    rows = M.golden_f7()
    tri, stats, _ = M.triangulate(rows)
    V, E, F, B, _ = M.topology(tri)
    assert B < 0.10 * E
    assert V > 0.95 * int((rows[7] > 0).sum())


def test_obj_round_trip(tmp_path):
    rows = M.with_merged()
    tri, _, _ = M.triangulate(rows)
    pos = rows[3:6].T.copy()
    pos[rows[7] < 0] = np.nan
    colors = (np.arange(3 * len(pos)) % 256).astype(np.uint8).reshape(-1, 3)
    nv, nf = mesh_io.write_obj(tmp_path / "m.obj", pos, colors, tri)
    v, c, f = mesh_io.read_obj(tmp_path / "m.obj")
    kept = np.flatnonzero(~np.isnan(pos[:, 0]))
    assert (nv, nf) == (len(kept), len(tri)) == (len(v), len(f))
    assert f.min() >= 0 and f.max() < len(v)
    np.testing.assert_allclose(v, pos[kept], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(c, colors[kept] / 255.0, atol=1e-5)
    np.testing.assert_array_equal(kept[f], np.asarray(tri, np.int64))
    text = (tmp_path / "m.obj").read_text().splitlines()
    assert text[0].startswith("v ") and len(text[0].split()) == 7 and text[-1].startswith("f ")


def test_obj_rejects_merged_corners(tmp_path):
    pos = np.zeros((3, 3), np.float32)
    pos[1] = np.nan
    with pytest.raises(ValueError):
        mesh_io.write_obj(tmp_path / "m.obj", pos, np.zeros((3, 3), np.uint8), [[0, 1, 2]])


def test_ply_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    pos = rng.random((50, 3)).astype(np.float32)
    pos[[3, 7]] = np.nan
    normals = rng.random((50, 3)).astype(np.float32)
    colors = rng.integers(0, 256, (50, 3)).astype(np.uint8)
    assert mesh_io.write_ply(tmp_path / "c.ply", pos, normals, colors) == 48
    d = mesh_io.read_ply(tmp_path / "c.ply")
    kept = np.flatnonzero(~np.isnan(pos[:, 0]))
    np.testing.assert_array_equal(np.stack([d["x"], d["y"], d["z"]], 1), pos[kept])
    np.testing.assert_array_equal(np.stack([d["nx"], d["ny"], d["nz"]], 1), normals[kept])
    np.testing.assert_array_equal(np.stack([d["red"], d["green"], d["blue"]], 1), colors[kept])


def test_struct_layouts():
    assert C.sizeof(_lib.MeshParams) == 12
    assert [f for f, _ in _lib.MeshParams._fields_] == ["neighbor_radius_factor", "max_angle_between_normals_deg",
                                                       "max_triangle_angle_deg"]
    assert C.sizeof(_lib.MeshStats) == 32
    assert _lib.MeshStats.umbrella_overflows.offset == 24
    p = _lib.MeshParams.defaults()
    assert (p.neighbor_radius_factor, p.max_angle_between_normals_deg, p.max_triangle_angle_deg) == (2.0, 90.0, 170.0)
    assert "sm_triangulate" in _lib.EXPORTED_SYMBOLS and "sm_default_mesh_params" in _lib.EXPORTED_SYMBOLS


def test_header_declares_the_call():
    from pathlib import Path
    h = (Path(__file__).resolve().parents[1] / "include" / "surfel_b200.h").read_text()
    assert "#define SM_MESH_MAX_UMBRELLA 16" in h and "int sm_triangulate(" in h
    assert h.count("sm_triangulate, sm_surfel_count") == 1   # a hand-off call between session pushes
    assert _lib.MESH_MAX_UMBRELLA == 16
