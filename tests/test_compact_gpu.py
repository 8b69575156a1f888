"""sm_compact on the GPU: the state after the call against the numpy restatement (tests/compact_walk.py), the
readers against the old handle's results through the map, the persistent mesh, sessions, the hand-off and the
use case (a session that stays under its surfel cap)."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import TransferToken
from tests import compact_walk as W
from tests.test_compact_host import state as hand_state
from tests.util import load_golden, params

pytestmark = pytest.mark.gpu

CAM = S.Camera.tum(320, 240)
# Rows an Integrate() writes the same on two handles that hold the same state; the smooth positions (rows 3-5) are
# sums of float atomics in arrival order (k_reg_accumulate), as tests/test_session_gpu.py's EXACT_ROWS excludes.
INTEGRATED_ROWS = (0, 1, 2, 6, 7, 8, 9, 10, 17, 18, 24)
SMOOTH_TOLERANCE = 1e-4   # metres
CAP = 400_000
K = 8
INV = W.INVALID


def make(cap=CAP, cam=CAM):
    return R.CUDASurfelReconstruction(cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


@pytest.fixture(scope="module")
def stream48():
    st = S.make_stream(CAM, 48, device="cuda")
    torch.cuda.synchronize()
    return st


def run(rec, st, first, last):
    pp, ip = params(CAM)
    return rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                          ip, first, last)


def assert_state(rec, rows_after, n_after, merges_after):
    rows, n, merges = rec.dump_state()
    assert n == n_after and merges == merges_after
    assert rec.surfels_size() == n_after and rec.surfel_count() == n_after - merges_after
    for r in W.CHECKED_ROWS:
        assert np.array_equal(rows[r].view(np.uint32), rows_after[r].view(np.uint32)), f"row {r}"


def assert_integrated_equal(ra, rb):
    for r in INTEGRATED_ROWS:
        assert np.array_equal(ra[r].view(np.uint32), rb[r].view(np.uint32)), f"row {r}"
    assert np.abs(ra[3:6] - rb[3:6]).max() <= SMOOTH_TOLERANCE


def compact_and_check(rec):
    rows, n, merges = rec.dump_state()
    want_rows, want_map, want_stats, want_merges = W.compact(rows, n, merges)
    stats, m = rec.compact(return_map=True)
    got_map = (m.cpu().numpy() & 0xFFFFFFFF).astype(np.uint32)
    assert np.array_equal(got_map, want_map)
    for k, v in want_stats.items():
        assert getattr(stats, k) == v, k
    assert_state(rec, want_rows, want_stats["slots_after"], want_merges)
    return rows, n, merges, want_map, stats


def hand_states():
    return {"alternating": (hand_state(8, range(1, 8, 2), {0: [1, 2, 4], 2: [0, 3], 6: [INV, 7, 6]}), 4),
            "boundary": (hand_state(2050, [1023, 1024, 2049], {1025: [1022, 1023, 1024, 1026], 0: [2049, 2048]}), 3),
            "all": (hand_state(6, range(6), {0: [1, 2]}), 6),
            "self_link": (hand_state(4, [2], {2: [2], 1: [2]}), 1)}


@pytest.mark.parametrize("name", ["f5", "f6", "f7", "alternating", "boundary", "all", "self_link"])
def test_state_equals_the_restatement(name):
    rec = make()
    if name.startswith("f"):
        g = load_golden()
        rows, merges = g[f"{name}_state"], int(g[f"{name}_counts"][1])
    else:
        rows, merges = hand_states()[name]
    rec.load_state(rows, merges)
    _, _, _, _, stats = compact_and_check(rec)
    assert stats.merged_removed > 0


def test_nothing_to_remove_is_a_no_op():
    g = load_golden()
    rec = make()
    rec.load_state(g["f4_state"], 0)
    buffers = R.make_cpu_buffers(CAP)
    token = TransferToken()
    rec.TransferDeltaToCPU(None, 10, buffers, token)
    before = rec.dump_state()
    launches = rec.lib.fn["kernel_launch_count"]()
    stats, m = rec.compact(return_map=True)
    assert rec.lib.fn["kernel_launch_count"]() == launches
    assert stats.slots_before == stats.slots_after == before[1] and stats.merged_removed == 0
    assert np.array_equal(m.cpu().numpy(), np.arange(before[1]))
    assert_state(rec, before[0], before[1], before[2])
    assert rec.TransferDeltaToCPU(None, 10, buffers, token).full_transfer == 0


def test_arguments():
    rec = make()
    rec.load_state(*hand_states()["alternating"])
    launches = rec.lib.fn["kernel_launch_count"]()
    short = torch.empty(7, dtype=torch.int32, device="cuda")
    status = rec.lib.fn["compact"](rec._h, None, C.c_void_p(short.data_ptr()), 7, None)
    assert status == _lib.SM_ERR_INVALID_ARGUMENT and rec.lib.fn["kernel_launch_count"]() == launches
    assert rec.lib.fn["compact"](None, None, None, 0, None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert rec.lib.fn["compact"](rec._h, None, None, 0, None) == _lib.SM_OK   # NULL map and stats
    assert rec.surfels_size() == 4 and rec.surfel_count() == 4


def test_free_running_stream_and_readers_commute(stream48):
    rec = make()
    first, last = stream48.integrated_range()
    run(rec, stream48, first, last)
    T = stream48.frame_T_global[last - 4]
    view = dict(width=CAM.width, height=CAM.height, fx=CAM.fx, fy=CAM.fy, cx=CAM.cx, cy=CAM.cy, near=0.1, far=20.0)
    tri_old, mstats_old = rec.triangulate()
    img_old = {k: v.cpu().numpy() for k, v in rec.render(T, **view).items()}
    pos_old, col_old = rec.export_vertices_host()
    mesh_img_old = {k: v.cpu().numpy() for k, v in rec.render_mesh(tri_old, T, **view).items()}
    _, n, merges, m, stats = compact_and_check(rec)
    print(f"48-frame stream: {n} slots, {merges} merged, {stats.links_dropped} links dropped")
    assert merges > 0
    # sm_triangulate: the same triangles in the same order, and the same stats
    tri_new, mstats_new = rec.triangulate()
    assert np.array_equal(tri_new.cpu().numpy(), W.remap_triangles(tri_old.cpu().numpy(), m).astype(np.int32))
    assert tri_new.shape[0] == tri_old.shape[0]
    for k in ("triangle_count", "vertices_meshed", "boundary_edges", "umbrella_overflows"):
        assert getattr(mstats_new, k) == getattr(mstats_old, k), k
    # sm_render_surfels: depth, colour and normal bit-exact, the index image through the map
    img_new = {k: v.cpu().numpy() for k, v in rec.render(T, **view).items()}
    for k in ("depth", "color", "normal"):
        assert np.array_equal(img_new[k].view(np.uint8), img_old[k].view(np.uint8)), k
    idx = img_old["index"]
    want = np.where(idx >= 0, m.astype(np.int64)[np.maximum(idx, 0)], -1)
    assert np.array_equal(img_new["index"], want)
    # sm_render_mesh over the remapped list
    mesh_img_new = {k: v.cpu().numpy() for k, v in rec.render_mesh(tri_new, T, **view).items()}
    for k in ("depth", "color", "normal"):
        assert np.array_equal(mesh_img_new[k].view(np.uint8), mesh_img_old[k].view(np.uint8)), k
    # sm_export_vertices: the non-NaN rows, in order
    pos_new, col_new = rec.export_vertices_host()
    live = ~np.isnan(pos_old[:, 0])
    assert np.array_equal(pos_new.view(np.uint32), pos_old[live].view(np.uint32))
    assert np.array_equal(col_new, col_old[live])


def test_persistent_mesh_is_carried_over(stream48):
    rec = make()
    first, last = stream48.integrated_range()
    run(rec, stream48, first, last - 6)
    rec.mesh_update()
    old = rec.mesh_triangles("all").cpu().numpy()
    _, _, _, m, stats = compact_and_check(rec)
    assert stats.mesh_remapped == 1
    assert np.array_equal(rec.mesh_triangles("all").cpu().numpy(), W.remap_triangles(old, m).astype(np.int32))
    u = rec.mesh_update()
    assert u.slots_changed == 0 and u.triangles_added == 0 and u.triangles_removed == 0
    run(rec, stream48, last - 6, last)
    u = rec.mesh_update()
    tri, mstats = rec.triangulate()
    assert np.array_equal(rec.mesh_triangles("all").cpu().numpy(), tri.cpu().numpy())
    assert u.mesh.triangle_count == mstats.triangle_count
    # frames since the last update merged slots the mesh still names: it is dropped and rebuilt
    run_more = make()
    run(run_more, stream48, first, last - 6)
    run_more.mesh_update()
    run(run_more, stream48, last - 6, last)
    stats = run_more.compact()
    assert stats.mesh_remapped == 0
    u = run_more.mesh_update()
    tri, _ = run_more.triangulate()
    assert u.full_sweep == 1 and np.array_equal(run_more.mesh_triangles("all").cpu().numpy(), tri.cpu().numpy())


def test_integration_continues_on_the_compacted_state(stream48):
    first, last = stream48.integrated_range()
    f = first + 20
    a = make()
    run(a, stream48, first, f)
    rows, n, merges = a.dump_state()
    want_rows, _, want_stats, want_merges = W.compact(rows, n, merges)
    a.compact()
    b = make()
    b.load_state(want_rows, want_merges)
    run(a, stream48, f, f + 1)
    run(b, stream48, f, f + 1)
    ra, na, ma = a.dump_state()
    rb, nb, mb = b.dump_state()
    assert na == nb and ma == mb
    assert_integrated_equal(ra, rb)


def near(a, b):
    """The float-atomic drift bound of tests/test_session_gpu.py."""
    return abs(int(a) - int(b)) <= 0.002 * max(a, b) + 5


@pytest.mark.parametrize("serial", [False, True], ids=["frame_graph", "serial"])
def test_session_compacts_between_pushes(stream48, serial):
    pp, ip = params(CAM)
    st = stream48
    p = 30
    a = make()
    if serial:
        a.enable_timings(True)
    compacted = {}
    with a.session(pp, ip, (CAM.width, CAM.height)) as s:
        for f in range(st.frame_count):
            status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            if f == p:
                rows, n, merges = a.dump_state()
                compacted["next"] = status.last_integrated_frame + 1
                compacted["want"] = W.compact(rows, n, merges)
                s.compact()
                want_rows, _, want_stats, want_merges = compacted["want"]
                assert_state(a, want_rows, want_stats["slots_after"], want_merges)
                assert a.surfel_count() == want_stats["slots_after"]
                assert np.count_nonzero(~np.isnan(a.export_vertices_host()[0][:, 0])) == a.surfel_count()
                with pytest.raises(_lib.SurfelError):
                    a.download_rasters()
            if f == p + 1:
                compacted["first"] = a.dump_state()
                a.download_rasters()   # an Integrate ran since
            if f > p:   # the counts stay consistent between pushes
                _, n_now, merges_now = a.dump_state()
                assert a.surfel_count() == n_now - merges_now
                assert np.count_nonzero(~np.isnan(a.export_vertices_host()[0][:, 0])) == a.surfel_count()
    want_rows, _, _, want_merges = compacted["want"]
    b = make()
    if serial:
        b.enable_timings(True)
    b.load_state(want_rows, want_merges)
    start = compacted["next"] - K // 2
    with b.session(pp, ip, (CAM.width, CAM.height), first_frame_index=start) as s:
        for f in range(start, st.frame_count):
            s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            if f == p + 1:
                rows_b, n_b, m_b = b.dump_state()
                rows_a, n_a, m_a = compacted["first"]
                assert n_a == n_b and m_a == m_b
                assert_integrated_equal(rows_a, rows_b)
    assert near(a.surfels_size(), b.surfels_size()) and near(a.surfel_count(), b.surfel_count())


def test_hand_off_after_compaction(stream48):
    rec = make()
    first, last = stream48.integrated_range()
    run(rec, stream48, first, last - 1)
    buffers = R.make_cpu_buffers(CAP)
    token = TransferToken()
    rec.TransferDeltaToCPU(None, last, buffers, token)
    rec.compact()
    stats = rec.TransferDeltaToCPU(None, last, buffers, token)
    assert stats.full_transfer == 1
    full = rec.TransferAllToCPU(None, last)
    n = rec.surfels_size()
    assert stats.surfel_count == n
    for k in R.BUFFER_NAMES:
        assert np.array_equal(buffers[k][:n].view(np.uint32), full[k][:n].view(np.uint32)), k
    with pytest.raises(_lib.SurfelError):
        rec.download_rasters()
    run(rec, stream48, last - 1, last)
    rec.download_rasters()


# The use case, on the 96-frame 320 x 240 synthetic stream. Measured on an H100 80GB HBM3 (700 W power limit): the
# plain session ends with 39 359 slots, 3 921 of them merged; with the cap at 37 399 (slots - merged / 2) the plain
# session drops new surfels (SM_ERR_CAPACITY), while compacting every 8 frames ends with 35 576 slots. Rendered depth
# against the ray-cast scene: median 1.47 / 1.48 mm and p95 16.70 / 16.69 mm (plain / compacting); the margin allowed
# is 25 % + 0.1 mm. The cap is set from the plain run, so the test holds for any stream.
def test_compacting_session_stays_under_the_cap():
    st = S.make_stream(CAM, 96, device="cuda")
    pp, ip = params(CAM)
    plain = make(cap=CAP)
    with plain.session(pp, ip, (CAM.width, CAM.height)) as s:
        for f in range(st.frame_count):
            s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
    size, live = plain.surfels_size(), plain.surfel_count()
    merged = size - live
    cap = size - merged // 2
    print(f"plain run: {size} slots, {live} live, {merged} merged; cap {cap}")
    assert merged > 0
    capped = make(cap=cap)
    with pytest.raises(_lib.SurfelError) as e:
        with capped.session(pp, ip, (CAM.width, CAM.height)) as s:
            for f in range(st.frame_count):
                s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
        capped.surfels_size()
    assert e.value.code == _lib.SM_ERR_CAPACITY
    kept = make(cap=cap)
    with kept.session(pp, ip, (CAM.width, CAM.height)) as s:
        for f in range(st.frame_count):
            s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            if f % 8 == 7:
                s.compact()
    assert kept.surfels_size() <= cap   # no SM_ERR_CAPACITY
    assert len(s.compactions) == st.frame_count // 8
    print(f"compacting run: {kept.surfels_size()} slots, {kept.surfel_count()} live")
    # the surface: rendered depth against the ray-cast scene, as tests/test_render_gpu.py measures it
    f = st.integrated_range()[1] - 4
    pose64 = torch.from_numpy(S.trajectory(st.frame_count)[f]).to("cuda")
    gt, _ = S._raycast(CAM, pose64, "cuda")
    errs = []
    for rec in (plain, kept):
        depth = rec.render(st.frame_T_global[f], CAM.width, CAM.height, CAM.fx, CAM.fy, CAM.cx, CAM.cy, near=0.1,
                           far=20.0, outputs=("depth",))["depth"].double()
        valid = torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0) & (depth > 0)
        err = (depth - gt)[valid].abs().cpu().numpy()
        errs.append((float(np.median(err)), float(np.percentile(err, 95))))
    print(f"median / p95 |d|: plain {errs[0]}, compacting {errs[1]}")
    assert errs[1][0] <= errs[0][0] * 1.25 + 1e-4 and errs[1][1] <= errs[0][1] * 1.25 + 1e-4


def test_session_policy_compacts_when_headroom_runs_low(stream48):
    pp, ip = params(CAM)
    probe = make()
    run(probe, stream48, *stream48.integrated_range())
    cap = probe.surfels_size() + 2000
    rec = make(cap=cap)
    with rec.session(pp, ip, (CAM.width, CAM.height), compact_when_free_below=0.2) as s:
        for f in range(stream48.frame_count):
            s.push(stream48.depth[f], stream48.color[f], stream48.global_T_frame[f], stream48.frame_T_global[f])
    assert len(s.compactions) > 0 and rec.surfels_size() <= cap
    with pytest.raises(ValueError):
        rec.session(pp, ip, (CAM.width, CAM.height), compact_when_free_below=1.5)
