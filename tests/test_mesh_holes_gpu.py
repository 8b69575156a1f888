"""sm_mesh_fill_holes on the GPU: bit-exact against the plain-C restatement (tests/hole_walk.c) on every mesh_walk
case, golden f7, the mesh of an integrated VGA stream and the persistent mesh of a session; argument and input
errors, the capacity protocol, independence from sm_mesh_update, the rendered coverage and the OBJ export."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, mesh_io, synthetic as S
from surfelmeshing_b200._lib import HoleParams, HoleStats, IntegrateParams, PreprocessParams
from tests import hole_walk as HW
from tests import mesh_walk as M
from tests.test_mesh_gpu import loaded, make, run_stream

pytestmark = pytest.mark.gpu

KS = (3, 4, 8, 16)
# (normal gate, largest triangle angle): the defaults, a gate narrow enough to reject loops of golden f7 (42 filled
# instead of 53 at K = 8), and an angle limit that rejects some (50 instead of 53)
GATES = ((90.0, 180.0), (10.0, 180.0), (30.0, 120.0))


def gpu_fill(rec, tri, K, normals=90.0, angle=180.0):
    f, stats = rec.fill_holes(tri, HoleParams(K, normals, angle))
    torch.cuda.synchronize()
    return f.cpu().numpy().astype(np.uint32), {k: int(getattr(stats, k)) for k, _ in HoleStats._fields_}


def assert_same(rec, rows, tri, ks=KS, gates=GATES):
    host_tri = tri.cpu().numpy().astype(np.uint32)
    for K in ks:
        for normals, angle in gates:
            want_f, want_s = HW.fill_holes(rows, host_tri, HoleParams(K, normals, angle))
            got_f, got_s = gpu_fill(rec, tri, K, normals, angle)
            assert got_s == want_s, (K, normals, angle)
            assert np.array_equal(got_f, want_f), (K, normals, angle)


def test_bit_equal_where_gate_angle_and_conflicts_decide():
    """The hand-built cases on which the normal gate, the angle test and rule H6 change the output."""
    cases = [(HW.tilted_corner_case(), [(8, 90.0, 180.0), (8, 40.0, 180.0)], (2, 0)),
             (HW.angle_case(), [(4, 90.0, 180.0), (4, 90.0, 120.0), (4, 90.0, 60.0)], (2, 2, 0))]
    rows, a, b, both = HW.conflict_case()
    cases.append(((rows, both), [(8, 180.0, 180.0), (8, 90.0, 180.0)], (0, 0)))
    cases.append(((rows, a), [(8, 180.0, 180.0)], (4,)))
    cases.append(((rows, b), [(8, 180.0, 180.0)], (2,)))
    conflicting = 0
    for (rows, tri), params, sizes in cases:
        rec = loaded(rows)
        t = torch.as_tensor(tri.astype(np.int32), device="cuda")
        for (K, normals, angle), size in zip(params, sizes):
            want_f, want_s = HW.fill_holes(rows, tri, HoleParams(K, normals, angle))
            got_f, got_s = gpu_fill(rec, t, K, normals, angle)
            assert got_s == want_s and np.array_equal(got_f, want_f), (K, normals, angle)
            assert len(got_f) == size
            conflicting += got_s["loops_conflicting"]
        rec.close()
    assert conflicting == 2


@pytest.mark.parametrize("name", sorted(M.CASES) + ["golden_f7"])
def test_bit_equal_to_restatement(name):
    rows = M.golden_f7() if name == "golden_f7" else M.CASES[name]()
    rec = loaded(rows)
    tri, _ = rec.triangulate()
    assert_same(rec, rows, tri)
    rec.close()


def test_bit_equal_on_an_integrated_stream():
    rec, _ = run_stream(S.Camera.tum(640, 480), 48)
    rows, _, _ = rec.dump_state()
    tri, _ = rec.triangulate()
    assert_same(rec, rows, tri)
    f, s = gpu_fill(rec, tri, 8)
    print(f"48-frame VGA stream, K = 8: {len(tri)} triangles, {s}")
    assert s["loops_filled"] > 0
    rec.close()


def session(updates_at):
    """Pushes a 24-frame QVGA stream through a session and hands the handle over after the pushes `updates_at`."""
    cam = S.Camera.tum(320, 240)
    st = S.make_stream(cam, 24, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    rec = make(cam)
    with rec.session(pp, IntegrateParams.defaults(), (cam.width, cam.height)) as s:
        for f in range(st.frame_count):
            s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            if f in updates_at:
                yield rec


def test_bit_equal_on_a_session_mesh_and_update_unchanged():
    """After several mesh_update()s, the fill of mesh_triangles("all") matches the restatement; a fill between two
    updates changes neither the next update's delta nor its equality with triangulate()."""
    gen = session((10, 14, 18))
    rec = next(gen)
    previous = None
    try:
        while True:
            rec.mesh_update()
            mesh = rec.mesh_triangles("all")
            rows, _, _ = rec.dump_state()
            if previous is not None:
                added = {tuple(t) for t in rec.mesh_triangles("added").cpu().numpy().tolist()}
                removed = {tuple(t) for t in rec.mesh_triangles("removed").cpu().numpy().tolist()}
                now = {tuple(t) for t in mesh.cpu().numpy().tolist()}
                assert added == now - previous and removed == previous - now
            tri, _ = rec.triangulate()
            assert torch.equal(tri, mesh)
            assert_same(rec, rows, mesh)   # fills between this update and the next one
            again = rec.mesh_update()
            assert again.triangles_added == 0 and again.triangles_removed == 0
            assert torch.equal(rec.mesh_triangles("all"), mesh)
            previous = {tuple(t) for t in mesh.cpu().numpy().tolist()}
            rec = next(gen)
    except StopIteration:
        pass
    rec.close()


def test_errors_write_nothing_and_capacity_protocol():
    rows, tri = HW.grid_mesh(8)
    rows = np.concatenate([rows, M.make_rows([[9.0, 9.0, 9.0]], (0, 0, 1), -1.0)], 1)   # slot 64: not present
    tri = HW.without(tri, [3 * 8 + 4])
    rec = loaded(rows)
    fn = rec.lib.fn["mesh_fill_holes"]
    p = HoleParams.defaults()
    stats = HoleStats()
    buf = torch.full((16, 3), -7, dtype=torch.int32, device="cuda")

    def call(t, params=p, out=buf, capacity=16, st=stats):
        t = torch.as_tensor(np.asarray(t, np.int32).reshape(-1, 3), device="cuda")
        status = fn(rec._h, None, C.byref(params) if params is not None else None, C.c_void_p(t.data_ptr()), len(t),
                    C.c_void_p(out.data_ptr()) if out is not None else None, capacity,
                    C.byref(st) if st is not None else None)
        torch.cuda.synchronize()
        return status

    launches = rec.lib.fn["kernel_launch_count"]()
    for bad in (HoleParams(2, 90, 180), HoleParams(17, 90, 180), HoleParams(8, 0, 180), HoleParams(8, 90, 181),
                HoleParams(8, float("nan"), 180)):
        assert call(tri, bad) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(tri, None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(tri, st=None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(tri, out=None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert rec.lib.fn["kernel_launch_count"]() == launches
    n = rows.shape[1]
    for t in ([[0, 1, n]], [[0, 1, 64]], [[0, 0, 1]], tri[:1]):
        assert call(np.concatenate([tri, t])) == _lib.SM_ERR_INVALID_ARGUMENT
        assert stats.triangles_added == 0
    assert rec.lib.fn["last_error"]() == b"sm_mesh_fill_holes: a directed edge occurs twice (the input must be " \
        b"edge-manifold and consistently oriented)"
    assert (buf == -7).all()
    # a count query, then a capacity one short, then enough
    assert call(tri, out=None, capacity=0) == _lib.SM_ERR_CAPACITY
    assert stats.triangles_added == 4 and stats.loops_filled == 1
    assert call(tri, capacity=3) == _lib.SM_ERR_CAPACITY and stats.triangles_added == 4
    assert rec.lib.fn["last_error"]() == b"sm_mesh_fill_holes: 4 triangles do not fit the capacity of 3"
    assert (buf == -7).all()
    assert call(tri) == _lib.SM_OK
    want, _ = HW.fill_holes(rows, tri)
    assert np.array_equal(buf[:4].cpu().numpy().astype(np.uint32), want) and (buf[4:] == -7).all()
    assert call(np.zeros((0, 3)), capacity=0) == _lib.SM_OK and stats.boundary_edges == 0
    rec.close()


def test_fill_covers_more_pixels_near_the_scene():
    cam = S.Camera.tum(640, 480)
    st = S.make_stream(cam, 48, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    rec = make(cam)
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                   IntegrateParams.defaults(), first, last)
    tri, _ = rec.triangulate()
    fill, stats = rec.fill_holes(tri)
    f = last - 4
    pose64 = torch.from_numpy(S.trajectory(st.frame_count)[f]).to("cuda")
    gt, _ = S._raycast(cam, pose64, "cuda")
    view = dict(width=cam.width, height=cam.height, fx=cam.fx, fy=cam.fy, cx=cam.cx, cy=cam.cy, near=0.1, far=20.0,
                unmeshed_surfels=False, outputs=("depth",))
    alone = rec.render_mesh(tri, st.frame_T_global[f], **view)["depth"].double()
    both = rec.render_mesh(torch.cat([tri, fill]), st.frame_T_global[f], **view)["depth"].double()
    gt_valid = torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0)
    before, after = alone > 0, both > 0
    assert not (before & ~after).any()
    new = gt_valid & after & ~before
    print(f"fill: {len(fill)} triangles ({stats.loops_filled} loops), {int(new.sum())} newly covered pixels")
    assert int((after & ~before).sum()) > 0
    # the band: the existing triangles' own error, 99th percentile, against the scene
    band = float(np.percentile((alone - gt)[gt_valid & before].abs().cpu().numpy(), 99))
    err = (both - gt)[new].abs().cpu().numpy()
    print(f"band {band * 1e3:.3f} mm; newly covered: median {np.median(err) * 1e3:.3f} mm, max {err.max() * 1e3:.3f} mm")
    assert float(np.percentile(err, 95)) <= band
    rec.close()


def test_obj_export(tmp_path):
    rec, _ = run_stream(S.Camera.tum(320, 240), 16, stream_id=3)
    rec.save_mesh_obj(tmp_path / "plain.obj")
    tri, _ = rec.triangulate()
    positions, colors = rec.export_vertices_host()
    mesh_io.write_obj(tmp_path / "before.obj", positions, colors, tri.cpu().numpy())
    assert (tmp_path / "plain.obj").read_bytes() == (tmp_path / "before.obj").read_bytes()
    fill, _ = rec.fill_holes(tri)
    rec.save_mesh_obj(tmp_path / "filled.obj", holes=HoleParams.defaults())
    _, _, faces = mesh_io.read_obj(tmp_path / "filled.obj")
    assert len(fill) > 0 and len(faces) == len(tri) + len(fill)
    rec.close()
