"""sm_mesh_simplify on the GPU: bit-exact against the plain-C restatement (tests/simplify_walk.c) on the hand-built
meshes, the sm_triangulate meshes of every mesh_walk case, golden f7 and an integrated stream (each with its fill),
over several targets and cost bounds; read-only behaviour, commutation with sm_compact, use of the output by
sm_mesh_fill_holes and sm_render_mesh, argument and input errors, the capacity protocol and the OBJ export."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, mesh_io, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import HoleParams, SimplifyParams, SimplifyStats
from tests import hole_walk as HW
from tests import mesh_walk as M
from tests import simplify_walk as SW
from tests.test_mesh_gpu import loaded, run_stream

pytestmark = pytest.mark.gpu


def param_sets(count):
    return [SimplifyParams.defaults(), SimplifyParams.defaults(max_cost=0.0),
            SimplifyParams.defaults(target_triangles=max(count // 2, 1)),
            SW.unbounded(target_triangles=max(count // 4, 1), max_rounds=64, max_angle_between_normals_deg=90.0,
                         max_triangle_angle_deg=170.0),
            SW.unbounded(target_triangles=max(count // 10, 1), max_rounds=64),
            SimplifyParams.defaults(max_cost=1e-4, max_angle_between_normals_deg=30.0, max_triangle_angle_deg=120.0),
            SimplifyParams.defaults(max_rounds=0)]


def gpu_simplify(rec, tri, params):
    out, stats = rec.simplify_mesh(tri, params)
    torch.cuda.synchronize()
    return out.cpu().numpy().astype(np.uint32), SW.stats_dict(stats)


def assert_same(rec, rows, tri, params_list=None):
    """tri: int32 CUDA tensor over rec's slots; rows: rec's state (rows 3-5 = smooth positions)."""
    host = tri.cpu().numpy().astype(np.uint32)
    for p in params_list or param_sets(len(host)):
        want, want_s = SW.simplify(rows, host, p)
        got, got_s = gpu_simplify(rec, tri, p)
        assert got_s == want_s, (p.target_triangles, p.max_cost, p.max_rounds)
        assert got.shape == want.shape and np.array_equal(got, want), (p.target_triangles, p.max_cost)


def with_fill(rec, tri):
    fill, _ = rec.fill_holes(tri)
    return torch.cat([tri, fill])


@pytest.mark.parametrize("name", sorted(SW.mesh_cases()))
def test_bit_equal_on_the_host_cases(name):
    rows, tri = SW.mesh_cases()[name]
    rec = loaded(rows)
    t = torch.as_tensor(tri.astype(np.int32), device="cuda")
    assert_same(rec, rows, t)
    if name in ("octahedron", "neck", "hub"):
        assert_same(rec, rows, t, [SW.unbounded(), SW.unbounded(max_cost=0.0, max_rounds=8)])
    rec.close()


@pytest.mark.parametrize("case", ["link_case", "repeat_case"])
def test_bit_equal_where_link_and_repeated_triangle_decide(case):
    """The meshes on which only rule (a), and only rule (c)'s repeated triangle, stops a collapse (see
    test_mesh_simplify_host.py): the kernel's own form of each test is held to the restatement where it decides."""
    rows, tri = getattr(SW, case)()
    rec = loaded(rows)
    t = torch.as_tensor(tri.astype(np.int32), device="cuda")
    params = [SW.unbounded(), SW.unbounded(max_rounds=1), SimplifyParams.defaults(max_cost=0.0),
              SimplifyParams.defaults()]
    assert_same(rec, rows, t, params)
    got, s = gpu_simplify(rec, t, SW.unbounded())
    if case == "link_case":
        assert s["collapses"] == 1 and 0 not in got and 2 in got
    else:
        assert s["collapses"] == 0 and np.array_equal(got, tri)
    rec.close()


@pytest.mark.parametrize("name", sorted(M.CASES) + ["golden_f7"])
def test_bit_equal_on_gpu_meshes(name):
    rows = M.golden_f7() if name == "golden_f7" else M.CASES[name]()
    rec = loaded(rows)
    tri, _ = rec.triangulate()
    assert_same(rec, rows, tri)
    assert_same(rec, rows, with_fill(rec, tri))
    rec.close()


def test_bit_equal_on_an_integrated_stream():
    rec, _ = run_stream(S.Camera.tum(320, 240), 24, stream_id=2)
    rows, _, _ = rec.dump_state()
    tri = with_fill(rec, rec.triangulate()[0])
    assert_same(rec, rows, tri)
    _, s = gpu_simplify(rec, tri, SimplifyParams.defaults())
    print(f"24-frame QVGA stream with its fill: {s}")
    assert s["collapses"] > 0
    rec.close()


def test_read_only():
    rec, _ = run_stream(S.Camera.tum(320, 240), 16, stream_id=3)
    rec.mesh_update()
    mesh = rec.mesh_triangles("all")
    before, n, merges = rec.dump_state()
    out, s = rec.simplify_mesh(mesh, SimplifyParams.defaults(target_triangles=len(mesh) // 4))
    assert s.collapses > 0
    after, n2, merges2 = rec.dump_state()
    keep = [r for r in range(before.shape[0]) if r not in (3, 4, 5)]
    assert (n2, merges2) == (n, merges)
    assert np.array_equal(before[keep].view(np.uint32), after[keep].view(np.uint32))
    assert torch.equal(rec.mesh_triangles("all"), mesh)
    again = rec.mesh_update()
    assert again.slots_changed == 0 and again.triangles_added == 0 and again.triangles_removed == 0
    rec.close()


def test_commutes_with_compaction():
    rec, _ = run_stream(S.Camera.tum(320, 240), 48)
    _, _, merges = rec.dump_state()
    assert merges > 0
    tri = with_fill(rec, rec.triangulate()[0])
    params = [SimplifyParams.defaults(), SimplifyParams.defaults(target_triangles=len(tri) // 4, max_cost=1e-4)]
    before = [rec.simplify_mesh(tri, p)[0] for p in params]
    _, m = rec.compact(return_map=True)
    mapped = R.remap_triangles(tri, m)
    assert len(mapped) == len(tri)
    for p, b in zip(params, before):
        after, _ = rec.simplify_mesh(mapped, p)
        assert torch.equal(after, R.remap_triangles(b, m))
    rec.close()


def depth_errors(depth, gt):
    covered = (depth > 0) & torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0)
    err = (depth - gt)[covered].abs().cpu().numpy()
    return int(covered.sum()), float(np.median(err)), float(np.percentile(err, 95))


def test_output_is_usable_downstream():
    cam = S.Camera.tum(640, 480)
    rec, st = run_stream(cam, 48)
    tri = with_fill(rec, rec.triangulate()[0])
    out, s = rec.simplify_mesh(tri, SW.unbounded(target_triangles=len(tri) // 4, max_rounds=64,
                                                 max_angle_between_normals_deg=90.0, max_triangle_angle_deg=170.0))
    assert s.triangles_out <= len(tri) // 4
    # sm_mesh_fill_holes takes the output (it is edge-manifold, consistently oriented, over present slots)
    fill, hs = rec.fill_holes(out)
    assert hs.boundary_edges == s.boundary_edges
    view = dict(width=cam.width, height=cam.height, fx=cam.fx, fy=cam.fy, cx=cam.cx, cy=cam.cy, near=0.1, far=20.0,
                unmeshed_surfels=False, outputs=("depth",))
    first, last = st.integrated_range()
    poses = S.trajectory(st.frame_count)
    for f in (first + 4, (first + last) // 2, last - 4):
        gt, _ = S._raycast(cam, torch.from_numpy(poses[f]).to("cuda"), "cuda")
        full = depth_errors(rec.render_mesh(tri, st.frame_T_global[f], **view)["depth"].double(), gt)
        simple = depth_errors(rec.render_mesh(out, st.frame_T_global[f], **view)["depth"].double(), gt)
        print(f"frame {f}: full {len(tri)} triangles: {full[0]} px, median {full[1] * 1e3:.3f} mm, p95 "
              f"{full[2] * 1e3:.3f} mm; simplified {len(out)}: {simple[0]} px, median {simple[1] * 1e3:.3f} mm, "
              f"p95 {simple[2] * 1e3:.3f} mm")
        # Bounds set from the first run on an H100 (the quarter-size mesh: the same covered pixels, median and p95
        # within 0.003 mm of the full mesh's on all three views, as the collapses the budget needs cost <= 6e-5 m^2,
        # mostly on planes). They leave 30x that margin for the stream's run-to-run variation, far below the full
        # mesh's own error (median 0.6 mm, p95 4.5 mm), so a collapse that moves the surface would show.
        assert simple[0] >= 0.95 * full[0]
        assert simple[1] <= full[1] + 1e-4 and simple[2] <= full[2] + 5e-4
    rec.close()


def test_errors_write_nothing_and_capacity_protocol():
    rows, tri = HW.grid_mesh(8)
    rows = np.concatenate([rows, M.make_rows([[9.0, 9.0, 9.0]], (0, 0, 1), -1.0)], 1)   # slot 64: not present
    rec = loaded(rows)
    fn = rec.lib.fn["mesh_simplify"]
    p = SimplifyParams.defaults(max_cost=0.0)
    stats = SimplifyStats()
    buf = torch.full((len(tri) + 8, 3), -7, dtype=torch.int32, device="cuda")
    src = torch.as_tensor(tri.astype(np.int32), device="cuda")

    def call(t=src, params=p, out=buf, capacity=None, st=stats, count=None):
        if not isinstance(t, torch.Tensor):
            t = torch.as_tensor(np.asarray(t, np.int32).reshape(-1, 3), device="cuda")
        status = fn(rec._h, None, C.byref(params) if params is not None else None,
                    C.c_void_p(t.data_ptr()) if t is not None else None, len(t) if count is None else count,
                    C.c_void_p(out.data_ptr()) if out is not None else None,
                    (len(out) if out is not None else 0) if capacity is None else capacity,
                    C.byref(st) if st is not None else None)
        torch.cuda.synchronize()
        return status

    want, want_s = SW.simplify(rows, tri, p)
    launches = rec.lib.fn["kernel_launch_count"]()
    for bad in (SimplifyParams.defaults(max_cost=-1.0), SimplifyParams.defaults(max_cost=float("nan")),
                SimplifyParams.defaults(max_angle_between_normals_deg=0.0),
                SimplifyParams.defaults(max_triangle_angle_deg=181.0),
                SimplifyParams.defaults(max_triangle_angle_deg=float("nan")),
                SimplifyParams.defaults(max_rounds=-1), SimplifyParams.defaults(max_rounds=1025)):
        assert call(params=bad) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(params=None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(st=None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(out=None, capacity=5) == _lib.SM_ERR_INVALID_ARGUMENT
    assert fn(rec._h, None, C.byref(p), None, 3, C.c_void_p(buf.data_ptr()), len(buf), C.byref(stats)) == \
        _lib.SM_ERR_INVALID_ARGUMENT
    assert call(out=src) == _lib.SM_ERR_INVALID_ARGUMENT                         # out is triangles
    assert call(out=buf, t=buf[2:2 + len(tri)]) == _lib.SM_ERR_INVALID_ARGUMENT  # out overlaps triangles
    assert call(count=1 << 28) == _lib.SM_ERR_INVALID_ARGUMENT
    assert rec.lib.fn["kernel_launch_count"]() == launches
    assert (buf == -7).all()
    n = rows.shape[1]
    for t in ([[0, 1, n]], [[0, 1, 64]], [[0, 0, 1]], tri[:1]):
        assert call(np.concatenate([tri, t])) == _lib.SM_ERR_INVALID_ARGUMENT
        assert stats.triangles_out == 0 and stats.stop_reason == 0
    assert rec.lib.fn["last_error"]() == b"sm_mesh_simplify: a directed edge occurs twice (the input must be " \
        b"edge-manifold and consistently oriented)"
    assert (buf == -7).all()
    # a count query, then a capacity one short, then enough
    assert call(out=None, capacity=0) == _lib.SM_ERR_CAPACITY and SW.stats_dict(stats) == want_s
    assert call(capacity=len(want) - 1) == _lib.SM_ERR_CAPACITY and stats.triangles_out == len(want)
    assert rec.lib.fn["last_error"]() == \
        f"sm_mesh_simplify: {len(want)} triangles do not fit the capacity of {len(want) - 1}".encode()
    assert (buf == -7).all()
    assert call() == _lib.SM_OK and SW.stats_dict(stats) == want_s
    got = buf[:len(want)].cpu().numpy().astype(np.uint32)
    assert np.array_equal(got, want) and (buf[len(want):] == -7).all()
    assert call(np.zeros((0, 3)), capacity=0) == _lib.SM_OK and stats.triangles_in == 0
    rec.close()


def test_obj_export(tmp_path):
    rec, _ = run_stream(S.Camera.tum(320, 240), 16, stream_id=3)
    rec.save_mesh_obj(tmp_path / "plain.obj")
    tri, _ = rec.triangulate()
    positions, colors = rec.export_vertices_host()
    mesh_io.write_obj(tmp_path / "before.obj", positions, colors, tri.cpu().numpy())
    assert (tmp_path / "plain.obj").read_bytes() == (tmp_path / "before.obj").read_bytes()
    p = SimplifyParams.defaults(target_triangles=len(tri) // 2, max_cost=1e-4)
    simple, _ = rec.simplify_mesh(with_fill(rec, tri), p)
    rec.save_mesh_obj(tmp_path / "simple.obj", holes=HoleParams.defaults(), simplify=p)
    v, _, faces = mesh_io.read_obj(tmp_path / "simple.obj")
    used = np.unique(simple.cpu().numpy())
    assert len(v) == len(used) and np.allclose(v, positions[used], rtol=1e-5, atol=1e-5)
    assert np.array_equal(used[faces], simple.cpu().numpy())
    rec.close()
