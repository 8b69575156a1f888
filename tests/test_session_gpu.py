"""Incremental sessions (sm_session_begin / push / end) against sm_stream_run on the same frames.

sm_stream_run always gets its transforms from sm_outlier_filter_transforms, which is what a session computes from
the pushed poses, so both sides consume identical inputs."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, TransferToken
from tests.util import check_state_invariants, count_mismatch

pytestmark = pytest.mark.gpu

CAM = S.Camera.tum(640, 480)
EXACT_ROWS = (0, 1, 2, 6, 7, 8, 9, 10, 17, 18)
TRANSFER_ROWS = (3, 4, 5, 7, 8, 9, 10, 18)   # the CUDASurfelBuffersCPU arrays, in R.BUFFER_NAMES order
CAP = 2_000_000
K = 8


@pytest.fixture(scope="module")
def vga():
    st = S.make_stream(CAM, 60, device="cuda")
    others = R.stream_outlier_filter_transforms(st.global_T_frame, st.frame_T_global, K, st.depth_scaling)
    torch.cuda.synchronize()
    return st, others


def params(cam=CAM):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    return pp, IntegrateParams.defaults()


def make(cam=CAM, lib=None):
    return R.CUDASurfelReconstruction(CAP, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=lib)


def frame(st, f, mode):
    if mode == "device":
        return st.depth[f], st.color[f]
    if mode == "pageable":
        return st.depth[f].cpu().numpy(), st.color[f].cpu().numpy()
    return st.depth[f].cpu().pin_memory(), st.color[f].cpu().pin_memory()


def run_session(rec, st, n, pp, ip, mode="device", between=None, size=(640, 480)):
    with rec.session(pp, ip, size) as s:
        for f in range(n):
            d, c = frame(st, f, mode)
            status = s.push(d, c, st.global_T_frame[f], st.frame_T_global[f])
            assert status.frames_pushed == f + 1
            if between:
                between(f, status)
    return s.stats


def run_stream(rec, st, others, n, pp, ip):
    return rec.stream_run(None, st.depth[:n], st.color[:n], st.global_T_frame[:n], st.frame_T_global[:n], others[:n],
                          pp, ip, K // 2, n - K // 2)


def assert_one_frame_equal(rec, ref):
    rows, n, _ = rec.dump_state()
    rows_ref, n_ref, _ = ref.dump_state()
    assert n == n_ref > 0
    for row in EXACT_ROWS:
        assert count_mismatch(rows[row], rows_ref[row]) == 0, f"row {row}"
    flags = rec.download_rasters()["new_surfel_flag_vector"]
    assert np.array_equal(flags, ref.download_rasters()["new_surfel_flag_vector"])


def near(a, b):
    """The float-atomic drift bound of tests/test_pyramid_gpu.py."""
    return abs(int(a) - int(b)) <= 0.002 * max(a, b) + 5


@pytest.mark.parametrize("mode", ["device", "pageable", "pinned"])
def test_one_integrated_frame(product, vga, mode):
    st, others = vga
    pp, ip = params()
    ref = make()
    run_stream(ref, st, others, 9, pp, ip)
    rec = make()
    stats = run_session(rec, st, 9, pp, ip, mode)
    assert stats.frames_integrated == 1
    assert stats.h2d_bytes == (0 if mode == "device" else 9 * 640 * 480 * (2 + 3))
    assert_one_frame_equal(rec, ref)


def test_serial_mode_with_timings(product, vga):
    st, others = vga
    pp, ip = params()
    ref = make()
    ref.enable_timings(True)
    run_stream(ref, st, others, 9, pp, ip)
    rec = make()
    rec.enable_timings(True)
    statuses = []
    stats = run_session(rec, st, 9, pp, ip, "pageable", between=lambda f, s: statuses.append(s.last_integrated_frame))
    assert statuses[-1] == 4, "serial pushes integrate p - K/2"
    assert stats.frames_integrated == 1
    assert_one_frame_equal(rec, ref)
    assert any(v > 0 for v in rec.GetTimings())


def test_whole_stream(product, vga):
    st, others = vga
    pp, ip = params()
    ref = make()
    want = run_stream(ref, st, others, 60, pp, ip)
    rec = make()
    last = []
    got = run_session(rec, st, 60, pp, ip, between=lambda f, s: last.append(s.last_integrated_frame))
    assert last[9] == -1   # the first integrated frame, K/2, needs frames up to K/2 + K/2 + 2
    assert last[10] == 4 and last[-1] == 59 - K // 2 - 2
    assert got.frames_integrated == want.frames_integrated == 52
    assert near(got.surfels_size, want.surfels_size) and near(got.surfel_count, want.surfel_count)
    check_state_invariants(*rec.dump_state()[:2])


@pytest.mark.parametrize("knob", ["pyramid_level", "median_filter_and_densify_iterations"])
def test_whole_stream_knobs(product, vga, knob):
    st, others = vga
    cam = CAM.scaled(1) if knob == "pyramid_level" else CAM
    pp, ip = params(cam)
    ref, rec = make(cam), make(cam)
    for r in (ref, rec):
        r.configure(knob, 1)
    want = run_stream(ref, st, others, 20, pp, ip)
    got = run_session(rec, st, 20, pp, ip, "pageable" if knob == "pyramid_level" else "device")
    assert got.frames_integrated == want.frames_integrated == 12
    assert near(got.surfels_size, want.surfels_size) and near(got.surfel_count, want.surfel_count)


def test_every_feature_allocates_and_frees_its_scratch(product, vga):
    """One handle creates the scratch of every feature on first use, then closes: the frame loop with host frames at a
    pyramid level, a session, both renders, both trackers, triangulation, the persistent mesh, hole filling and the
    delta transfer's staging. A second handle does the same after the first one's frees, with sm_mesh_update first,
    which creates the meshing scratch without sm_triangulate."""
    st, others = vga
    cam = CAM.scaled(1)
    pp, ip = params(cam)
    n = 20
    depth, color = st.depth[:n].cpu().pin_memory(), st.color[:n].cpu().pin_memory()
    f = n - 1
    live_depth, live_color = st.depth[f, ::2, ::2].contiguous(), st.color[f, ::2, ::2].contiguous()
    view = (st.frame_T_global[f], cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    for update_first in (False, True):
        rec = make(cam)
        rec.configure("pyramid_level", 1)
        stats = rec.stream_run(None, depth, color, st.global_T_frame[:n], st.frame_T_global[:n], others[:n], pp, ip,
                               K // 2, n - K // 2)
        assert stats.frames_integrated == n - K
        assert run_session(rec, st, 12, pp, ip, "pinned").frames_integrated == 12 - K
        rec.track(live_depth, st.global_T_frame[f], pp=pp)
        rec.track_rgbd(live_depth, live_color, st.global_T_frame[f], pp=pp)
        assert int((rec.render(*view)["index"] >= 0).sum()) > 0
        if update_first:
            rec.mesh_update()
        triangles, _ = rec.triangulate()
        if not update_first:
            rec.mesh_update()
        assert len(triangles) > 0
        rec.fill_holes(triangles)
        rec.render_mesh(triangles, *view)
        buffers, token = R.make_cpu_buffers(rec.surfels_size()), TransferToken()
        assert rec.TransferDeltaToCPU(None, f, buffers, token).full_transfer == 1
        rec.Regularize(None, f, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, 1)
        assert rec.TransferDeltaToCPU(None, f, buffers, token).full_transfer == 0   # through the staging list
        rec.close()
    torch.cuda.synchronize()


def test_hand_off_between_pushes(product, vga):
    st, others = vga
    pp, ip = params()
    rec = make()
    persistent = R.make_cpu_buffers(CAP)
    token = TransferToken()
    checked = []

    def between(f, status):
        if f < 20 or f % 5 != 0:
            return
        full = rec.TransferAllToCPU(None, f)
        rows, n, merges = rec.dump_state()
        assert full["surfel_count"] == n
        for name, row in zip(R.BUFFER_NAMES, TRANSFER_ROWS):
            assert count_mismatch(full[name][:n], rows[row]) == 0, (f, name)
        rec.TransferDeltaToCPU(None, f, persistent, token)
        torch.cuda.synchronize()
        for name in R.BUFFER_NAMES:
            assert count_mismatch(persistent[name][:n], full[name][:n]) == 0, (f, name)
        # The counts are those after Integrate(status.last_integrated_frame). Every merge counted so far is applied
        # in the rows (radius_squared -1); the front half of the step the push launched has already decided the
        # next frame's merges, which must not show yet.
        surfel_count = rec.surfel_count()
        assert merges == int(np.count_nonzero(rows[7] < 0)), (f, merges)
        assert surfel_count == n - merges
        positions = torch.empty(3 * n, dtype=torch.float32, device="cuda")
        colors = torch.empty(3 * n, dtype=torch.uint8, device="cuda")
        rec.ExportVertices(None, positions, colors)
        torch.cuda.synchronize()
        assert int((~torch.isnan(positions[0::3])).sum()) == surfel_count   # APP/main.cc:150
        # against sm_stream_run up to the same frame (its last step has no next frame)
        ref = make()
        want = run_stream(ref, st, others, status.last_integrated_frame + 1 + K // 2, pp, ip)
        ref_rows, ref_n, ref_merges = ref.dump_state()
        assert ref_merges == int(np.count_nonzero(ref_rows[7] < 0))
        assert near(n, want.surfels_size), (f, n, want.surfels_size)
        assert near(surfel_count, want.surfel_count), (f, surfel_count, want.surfel_count)
        checked.append(f)

    run_session(rec, st, 36, pp, ip, between=between)
    assert checked == [20, 25, 30, 35]


def test_ordering_of_calls_on_the_stream(product, vga):
    st, others = vga
    pp, ip = params()
    rec = make()
    with rec.session(pp, ip, (640, 480)) as s:
        for f in range(20):
            s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
        rows, n, _ = rec.dump_state()
        bufs = R.make_cpu_buffers(n, pinned=True)
        count = C.c_uint64()
        rec.lib.call("transfer_all_to_cpu", rec._h, R._stream_handle(None), 19,
                     *[bufs[k].ctypes.data_as(C.c_void_p) for k in R.BUFFER_NAMES], C.byref(count))
        s.push(st.depth[20], st.color[20], st.global_T_frame[20], st.frame_T_global[20])
        torch.cuda.synchronize()
        assert count.value == n
        for name, row in zip(R.BUFFER_NAMES, TRANSFER_ROWS):
            assert count_mismatch(bufs[name][:n], rows[row]) == 0, name


def smooth_equal_fraction(a, b):
    """Fraction of the common slots whose smooth position (rows 3-5) is bit-equal."""
    n = min(a.shape[1], b.shape[1])
    same = np.all(a[3:6, :n].view(np.uint32) == b[3:6, :n].view(np.uint32), axis=0)
    return float(same.mean())


def test_regularize_between_pushes(product, vga):
    """sm_regularize between pushes of a frame-graph session acts on the state of status.last_integrated_frame, and
    the next step starts from the smooth buffers and the window it left. Compared with a serial session (one frame
    integrated per push, nothing of the next frame in flight) given the same Regularize() calls at the same newest
    integrated frames; a serial session without them is the control that shows what the calls change."""
    st, others = vga
    pp, ip = params()
    regularize_at = (12, 15)

    def run(serial, regularize):
        rec = make()
        if serial:
            rec.enable_timings(True)
        done = set()

        def between(f, status):
            frame = status.last_integrated_frame
            if regularize and frame in regularize_at and frame not in done:
                done.add(frame)
                rec.Regularize(None, frame, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors,
                               ip.regularization_frame_window_size)
                rows, n, _ = rec.dump_state()
                stamps = rows[18].view(np.uint32)
                detach = (rows[24].view(np.uint32) >> np.uint32(24)) == np.uint32(1)
                assert np.array_equal(rows[15].view(np.uint32),
                                      stamps | np.where(detach, np.uint32(0x80000000), np.uint32(0)))
                check_state_invariants(rows, n)

        stats = run_session(rec, st, 22, pp, ip, between=between)
        assert stats.frames_integrated == 14
        assert not regularize or done == set(regularize_at)
        rows, n, _ = rec.dump_state()
        check_state_invariants(rows, n)
        return rows

    graph = run(False, True)
    serial = run(True, True)
    control = run(True, False)
    same, ctrl = smooth_equal_fraction(graph, serial), smooth_equal_fraction(graph, control)
    assert same >= 0.9 and ctrl <= same - 0.05, (same, ctrl)


def test_rejected_calls(product, vga):
    st, others = vga
    pp, ip = params()
    ref = make()
    run_stream(ref, st, others, 9, pp, ip)
    rec = make()
    h, lib = rec._h, rec.lib
    bad = _lib.SM_ERR_INVALID_ARGUMENT
    assert lib.fn["session_push"](h, None, 0, None, 0, 0, None, None, None) == bad   # no session
    assert lib.fn["session_end"](h, None) == bad
    g, l = (np.ascontiguousarray(a[0].reshape(12)) for a in (st.global_T_frame, st.frame_T_global))
    with rec.session(pp, ip, (640, 480)) as s:
        for f in range(3):
            s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
        stream = R._stream_handle(None)
        assert lib.fn["integrate"](h, stream, 0, C.byref(ip), None, 0, None, 0, None, 0, None, 0, None, None) == bad
        assert b"session" in lib.fn["last_error"]()
        assert lib.fn["preprocess"](h, stream, C.byref(pp), None, 0, None, None, None, None, 0, None, 0, None, 0) == bad
        assert lib.fn["reset"](h, stream) == bad
        assert lib.fn["load_state"](h, stream, None, 0, 0, 0) == bad
        desc = _lib.StreamDesc(640, 480, 9, 0, st.depth.data_ptr(), st.color.data_ptr(), 0, 0, 0)
        assert lib.fn["stream_run"](h, stream, C.byref(desc), C.byref(pp), C.byref(ip), 4, 5, None) == bad
        assert lib.fn["configure"](h, b"pyramid_level", 0.0) == bad
        assert lib.fn["enable_timings"](h, 1) == bad
        assert lib.fn["timeline_enable"](h, 4) == bad
        assert lib.fn["session_begin"](h, stream, C.byref(pp), C.byref(ip), 640, 480, 0) == bad
        # bad pushes are not consumed
        d, c = st.depth[3], st.color[3]
        status = _lib.SessionStatus()
        gp, lp = g.ctypes.data_as(C.c_void_p), l.ctypes.data_as(C.c_void_p)
        assert lib.fn["session_push"](h, d.data_ptr(), 100, c.data_ptr(), 640 * 3, 0, gp, lp, C.byref(status)) == bad
        assert lib.fn["session_push"](h, None, 1280, c.data_ptr(), 640 * 3, 0, gp, lp, C.byref(status)) == bad
        assert lib.fn["session_push"](h, d.data_ptr(), 1280, c.data_ptr(), 640 * 3, 0, None, lp, C.byref(status)) == bad
        for f in range(3, 9):
            status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
        assert status.frames_pushed == 9
    assert s.stats.frames_integrated == 1
    assert_one_frame_equal(rec, ref)
    # sm_destroy with an open session drains it; a new handle then runs normally
    other = make()
    session = other.session(pp, ip, (640, 480))
    for f in range(12):
        session.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
    other.close()
    fresh = make()
    assert run_stream(fresh, st, others, 9, pp, ip).frames_integrated == 1
    assert_one_frame_equal(fresh, ref)


def test_against_reference(product, reference, vga):
    st, others = vga
    pp, ip = params()
    oracle = make(lib=reference)
    want = run_stream(oracle, st, others, 20, pp, ip)
    got = run_session(make(), st, 20, pp, ip)
    assert got.frames_integrated == want.frames_integrated == 12
    assert abs(int(got.surfels_size) - int(want.surfels_size)) <= 0.01 * want.surfels_size
