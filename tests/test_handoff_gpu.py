"""The hand-off of the surfel cloud to the CPU and the viewer: sm_update_visualization_buffers, sm_export_vertices and
sm_transfer_all_to_cpu bit for bit against the reference's kernels and against the float64 restatements of
tests/handoff_walk.py, and sm_transfer_delta_to_cpu through its record path: after every call the arrays equal a
fresh full transfer, and the statistics equal what the restated selection predicts."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, TransferToken
from tests import handoff_walk as HW
from tests.util import other_frames

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD        # a NaN no kernel writes: the words a call leaves alone keep it
CAM = S.Camera.tum(320, 240)
K = 8
GOLDEN_FRAMES = (4, 5, 6, 7)
ALL_BUFFERS = ("vertex", "neighbor", "normal")


def grid_pass():
    """Slots one grid-stride pass of the hand-off kernels covers: multiProcessorCount x 8 blocks x 256 threads."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256


def make(cap, lib=None):
    return R.CUDASurfelReconstruction(cap, CAM.width, CAM.height, CAM.fx, CAM.fy, CAM.cx, CAM.cy, lib=lib)


@pytest.fixture(scope="module")
def big():
    n = grid_pass() + 4099
    assert n % 32 != 0
    rows, merges = HW.constructed_state(n)
    return rows, merges


def golden_state(golden, f):
    return golden[f"f{f}_state"], int(golden[f"f{f}_counts"][1])


def state_cases(golden, big):
    return [(f"golden_f{f}",) + golden_state(golden, f) for f in GOLDEN_FRAMES] + [("constructed",) + big]


# ---- visualisation buffers ---------------------------------------------------------------------------------------
def viz(rec, n, point_size=4, frame=4000, window=30, tri=0xFFFFFFFF, mesh=0, flags=(0, 0, 0, 0),
        which=ALL_BUFFERS, extra=37):
    """One sm_update_visualization_buffers into sentinel-filled buffers `extra` slots longer than n; returns the
    three buffers (None where not passed) as u32 arrays."""
    def buf(width, name):
        if name not in which:
            return None
        return torch.full(((n + extra) * width,), SENTINEL, dtype=torch.int32, device="cuda")
    v, nb, nv = buf(point_size, "vertex"), buf(8, "neighbor"), buf(6, "normal")
    rec.UpdateVisualizationBuffers(None, frame, tri, mesh, window, *flags, vertex_buffer=v, neighbor_index_buffer=nb,
                                   normal_vertex_buffer=nv, point_size_in_floats=point_size)
    torch.cuda.synchronize()
    return [t.cpu().numpy().view(np.uint32) if t is not None else None for t in (v, nb, nv)]


def check_viz_restated(bufs, rows, point_size=4, frame=4000, window=30, tri=0xFFFFFFFF, mesh=0, flags=(0, 0, 0, 0),
                       counts=None):
    """Hold the three buffers to the restatement on `rows`: bit-exact where no approximate rcp / sqrt is involved;
    colours one count off at most, and only within HW.NEAR of a truncation point; end points within 2 ulps of the
    scale of their terms. Unwritten words keep the sentinel."""
    n = rows.shape[1]
    v, nb, nv = bufs
    mode = HW.viz_mode(*flags)
    if v is not None:
        v = v.reshape(-1, point_size)
        assert np.all(v[n:] == SENTINEL) and np.all(v[:n, 4:] == SENTINEL), "words beyond a vertex were written"
        want, close = HW.vertex_buffer(rows, frame, window, tri, mesh, mode)
        assert np.array_equal(v[:n, :3], want[:, :3]), "vertex positions"
        got_c, want_c = v[:n, 3], want[:, 3]
        diff = got_c != want_c
        far = diff & ~close
        assert not far.any(), (mode, np.flatnonzero(far)[:10], got_c[far][:10], want_c[far][:10])
        for shift in (0, 8, 16, 24):
            a = ((got_c[diff] >> shift) & 0xFF).astype(np.int64)
            b = ((want_c[diff] >> shift) & 0xFF).astype(np.int64)
            assert np.all(np.abs(a - b) <= (1 if shift < 24 else 0)), (mode, shift)
        if counts is not None:
            counts["near"] = counts.get("near", 0) + int(close.sum())
            counts["one_count"] = counts.get("one_count", 0) + int(diff.sum())
    if nb is not None:
        nb = nb.reshape(-1, 8)
        assert np.all(nb[n:] == SENTINEL)
        assert np.array_equal(nb[:n], HW.neighbor_segments(rows)), "neighbour segments"
    if nv is not None:
        nv = nv.reshape(-1, 6)
        assert np.all(nv[n:] == SENTINEL)
        _, end, scale = HW.normal_end_points(rows)
        assert np.array_equal(nv[:n, :3], rows[3:6].view(np.uint32).T), "normal segment starts"
        got = nv[:n, 3:].view(np.float32).astype(np.float64)
        finite = np.isfinite(end)
        tol = 2 * np.spacing(scale.astype(np.float32)).astype(np.float64)
        assert np.all(np.abs(got[finite] - end[finite]) <= tol[finite]), "normal end points beyond 2 ulps"
        nan = np.isnan(end)
        assert np.all(np.isnan(got[nan]))
        inf = ~finite & ~nan
        assert np.array_equal(got[inf], end[inf])


def viz_cases(rows, n):
    """(point_size, frame, window, tri, mesh, flags, which) over the parameter edges."""
    creation = rows[17].view(np.uint32)
    stamps = rows[18].view(np.uint32)
    s = int(np.median(creation))
    frame = int(stamps.max()) + 2
    cases = []
    for bits in range(16):      # every flag combination, all three buffers
        cases.append((4, frame, 30, s, n // 2, tuple((bits >> k) & 1 for k in range(4)), ALL_BUFFERS))
    for mode_flags in [(0, 0, 0, 0), (1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1)]:
        cases.append((7, frame, 30, s, n // 3, mode_flags, ("vertex",)))
    for tri in (s - 1, s, s + 1, 0, 0xFFFFFFFF):
        for mesh in (0, 1, n // 2 - 1, n // 2, n // 2 + 1, n - 1, n, n + 1, 0xFFFFFFFF):
            cases.append((4, frame, 30, tri, mesh, (0, 0, 0, 0), ("vertex",)))
    # every age from -2 to max_age + 2 in the two age modes
    lo, hi = int(stamps.min()), int(stamps.max())
    for window in (1, 2, 30, HW.INT_MAX):
        reach = min(window, 40) if window < HW.INT_MAX else 3
        frames = range(lo - 2, hi + reach + 3) if hi - lo < 200 else [frame, lo + window + 2 if window < 4000 else frame]
        for f in frames:
            cases.append((4, f, window, s, n, (1, 0, 0, 0), ("vertex",)))
    lo_c, hi_c = int(creation.min()), int(creation.max())
    frames = set()
    for age in (-2, -1, 0, 1, 2, 3, 1500, 2998, 2999, 3000, 3001, 3002):
        frames |= {lo_c + age, hi_c + age} if hi_c - lo_c >= 200 else set(range(lo_c + age, hi_c + age + 1))
    for f in sorted(frames):
        cases.append((4, f, 30, s, n, (0, 1, 0, 0), ("vertex",)))
    for which in (("vertex",), ("neighbor",), ("normal",)):   # each buffer alone
        cases.append((4, frame, 30, s, n, (0, 0, 1, 0), which))
    return cases


def test_state_ages_reach_every_edge(big):
    """The constructed state alone reaches every age of both ramps at one frame index."""
    rows, _ = big
    for row in (17, 18):
        a = HW.ages(rows[row].view(np.uint32)[rows[7] >= 0], 4000)
        assert np.isin(np.arange(-2, HW.CREATION_MAX_AGE + 3), a).all()


def all_viz_cases(case, rows):
    n = rows.shape[1]
    cases = viz_cases(rows, n)
    if case == "constructed":   # one frame index reaches every age: sweep the window instead
        cases += [(4, 4000, w, 0, 0, (1, 0, 0, 0), ("vertex",)) for w in (1, 2, 30, 3000, HW.INT_MAX)]
        cases += [(4, 4000, 30, 3000, n // 2, (0, 1, 0, 0), ALL_BUFFERS)]
    return cases


@pytest.mark.parametrize("case", ["golden_f4", "golden_f5", "golden_f6", "golden_f7", "constructed"])
def test_visualization_buffers_against_the_reference(product, reference, golden, big, case):
    _, rows, merges = [c for c in state_cases(golden, big) if c[0] == case][0]
    n = rows.shape[1]
    recs = []
    for lib in (product, reference):
        rec = make(n + 64, lib)
        rec.load_state(rows, merges)
        recs.append(rec)
    for point_size, frame, window, tri, mesh, flags, which in all_viz_cases(case, rows):
        args = dict(point_size=point_size, frame=frame, window=window, tri=tri, mesh=mesh, flags=flags)
        got = viz(recs[0], n, which=which, **args)
        want = viz(recs[1], n, which=which, **args)
        for label, g, w in zip(ALL_BUFFERS, got, want):
            assert (g is None) == (w is None)
            if g is not None:   # whole buffers: sentinel words included, NaN bit patterns included
                bad = np.flatnonzero(g != w)
                assert bad.size == 0, (case, label, args, bad[:8], g[bad[:8]], w[bad[:8]])
    for rec in recs:
        rec.close()


@pytest.mark.parametrize("case", ["golden_f4", "golden_f5", "golden_f6", "golden_f7", "constructed"])
def test_visualization_buffers_against_the_restatement(product, golden, big, case):
    _, rows, merges = [c for c in state_cases(golden, big) if c[0] == case][0]
    n = rows.shape[1]
    rec = make(n + 64)
    rec.load_state(rows, merges)
    counts = {}
    for point_size, frame, window, tri, mesh, flags, which in all_viz_cases(case, rows):
        args = dict(point_size=point_size, frame=frame, window=window, tri=tri, mesh=mesh, flags=flags)
        check_viz_restated(viz(rec, n, which=which, **args), rows, counts=counts, **args)
    if case == "constructed":
        assert counts["near"] > 1000   # the crossings of the ramps were reached
    print(f"\n{case}: colours within NEAR of a truncation point {counts.get('near', 0)}, one count off "
          f"{counts.get('one_count', 0)}")
    rec.close()


def test_visualization_rejections_write_nothing(product, golden):
    rows, merges = golden_state(golden, 7)
    n = rows.shape[1]
    rec = make(n + 64)
    rec.load_state(rows, merges)
    p = _lib.VisualizationParams(10, 0, 0, 30, 4, 0, 0, 0, 0)
    bufs = [torch.full(((n + 8) * w,), SENTINEL, dtype=torch.int32, device="cuda") for w in (8, 8, 6)]
    vertex, nb, nv = bufs
    misaligned = nb[1:]     # 4 bytes past a 16-byte boundary
    ptr = lambda t: C.c_void_p(t.data_ptr())
    status = product.fn["update_visualization_buffers"](rec._h, None, C.byref(p), ptr(vertex), ptr(misaligned), ptr(nv))
    assert status == _lib.SM_ERR_INVALID_ARGUMENT
    for size in (0, 1, 3):
        p.point_size_in_floats = size
        status = product.fn["update_visualization_buffers"](rec._h, None, C.byref(p), ptr(vertex), ptr(nb), ptr(nv))
        assert status == _lib.SM_ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    for t in bufs:
        assert bool((t == SENTINEL).all()), "a rejected call wrote a buffer"
    rec.close()


# ---- export and full transfer ------------------------------------------------------------------------------------
def export(rec, n, extra=11):
    pos = torch.full((3 * (n + extra),), SENTINEL, dtype=torch.int32, device="cuda")
    col = torch.full((3 * (n + extra),), 0xA5, dtype=torch.uint8, device="cuda")
    rec.ExportVertices(None, pos, col)
    torch.cuda.synchronize()
    pos, col = pos.cpu().numpy().view(np.uint32), col.cpu().numpy()
    assert np.all(pos[3 * n:] == SENTINEL) and np.all(col[3 * n:] == 0xA5), "export wrote past surfels_size()"
    return pos[:3 * n].reshape(n, 3), col[:3 * n].reshape(n, 3)


def host_arrays(n, pinned, extra=13):
    bufs = R.make_cpu_buffers(n + extra, pinned=pinned)
    for k in R.BUFFER_NAMES:
        bufs[k].view(np.uint32)[:] = SENTINEL
    return bufs


def full_transfer(rec, n, pinned=False, extra=13):
    bufs = host_arrays(n, pinned, extra)
    out = rec.TransferAllToCPU(None, 0, bufs)
    assert out["surfel_count"] == n
    for k in R.BUFFER_NAMES:
        assert np.all(bufs[k].view(np.uint32)[n:] == SENTINEL), "the transfer wrote past surfels_size()"
    return np.stack([bufs[k][:n].view(np.uint32) for k in R.BUFFER_NAMES])


@pytest.mark.parametrize("case", ["golden_f4", "golden_f5", "golden_f6", "golden_f7", "constructed"])
def test_export_and_transfer_against_the_reference(product, reference, golden, big, case):
    name, rows, merges = [c for c in state_cases(golden, big) if c[0] == case][0]
    n = rows.shape[1]
    results = []
    for lib in (product, reference):
        rec = make(n + 64, lib)
        rec.load_state(rows, merges)
        pos, col = export(rec, n)
        arrays = [full_transfer(rec, n, pinned) for pinned in (False, True)]
        results.append((pos, col, arrays))
        rec.close()
    (pos, col, arrays), (pos_r, col_r, arrays_r) = results
    assert np.array_equal(pos, pos_r) and np.array_equal(col, col_r)
    for a, b in zip(arrays + arrays_r, arrays[:1] * 4):
        assert np.array_equal(a, b)
    want_pos, want_col = HW.export_vertices(rows)
    assert np.array_equal(pos, want_pos) and np.array_equal(col, want_col)
    assert np.array_equal(arrays[0], rows[list(HW.TRANSFER_ROWS)].view(np.uint32))


def test_hand_off_reads_the_live_smooth_positions(product, golden):
    """After a Regularize() that moves surfels, the visualisation buffers, the export and the delta transfer are taken
    first; only then the full transfer and the dump, which refresh the rows 3-5 mirror. All agree with those rows."""
    rows0, merges = golden_state(golden, 7)
    n = rows0.shape[1]
    rec = make(n + 64)
    rec.load_state(rows0, merges)
    arrays, token = host_arrays(n, False), TransferToken()
    rec.TransferDeltaToCPU(None, 7, arrays, token)
    ip = IntegrateParams.defaults()
    for _ in range(3):      # window start 6: the surfels of frames 6 and 7 move, 4/5 of the cloud
        rec.Regularize(None, 7, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, 1)
    flags = (0, 0, 0, 1)
    bufs = viz(rec, n, frame=8, window=30, tri=0xFFFFFFFF, mesh=0, flags=flags)
    pos, col = export(rec, n)
    stats = rec.TransferDeltaToCPU(None, 8, arrays, token)
    assert stats.full_transfer == 0 and stats.changed_count == int((rows0[18].view(np.int32) >= 6).sum())
    full = full_transfer(rec, n)
    rows, n2, _ = rec.dump_state()
    assert n2 == n
    moved = np.any(rows[3:6] != rows0[3:6], axis=0)
    assert moved.sum() > n // 4, "the regularisation moved too few surfels to tell the mirror from the records"
    check_viz_restated(bufs, rows, frame=8, window=30, tri=0xFFFFFFFF, mesh=0, flags=flags)
    want_pos, want_col = HW.export_vertices(rows)
    assert np.array_equal(pos, want_pos) and np.array_equal(col, want_col)
    assert np.array_equal(np.stack([arrays[k][:n].view(np.uint32) for k in R.BUFFER_NAMES]), full)
    assert np.array_equal(full, rows[list(HW.TRANSFER_ROWS)].view(np.uint32))
    rec.close()


# ---- the delta transfer ------------------------------------------------------------------------------------------
class Copy:
    """One set of CUDASurfelBuffersCPU arrays, its token, and the operations issued since the token was filled."""

    def __init__(self, cap, pinned=False):
        self.arrays = host_arrays(cap, pinned, extra=0)
        self.token = TransferToken()
        self.ops = []


class Ledger:
    """What the delta transfers reached: the largest record count, the merge-only selections, the paths taken."""

    def __init__(self):
        self.largest = 0
        self.merge_only = 0
        self.paths = {"record": 0, "fallback": 0, "eight_ninths": 0}


def delta(rec, copy, frame, ledger, expect=None):
    """sm_transfer_delta_to_cpu into `copy`, then hold the arrays to a fresh full transfer and the statistics to the
    restated selection. `expect` = "fallback" for a full transfer decided before the selection (a token that does not
    apply, or a window start <= 0); otherwise the restatement decides between the record path and the 9/8 fallback."""
    cap = len(copy.arrays[R.BUFFER_NAMES[0]])
    before = {k: copy.arrays[k].view(np.uint32).copy() for k in R.BUFFER_NAMES}
    token_count, token_epoch = int(copy.token.surfel_count), int(copy.token.epoch)
    threshold = HW.stamp_threshold(copy.ops)
    stats = rec.TransferDeltaToCPU(None, frame, copy.arrays, copy.token)
    rows, n, _ = rec.dump_state()
    full = full_transfer(rec, n)
    got = np.stack([copy.arrays[k][:n].view(np.uint32) for k in R.BUFFER_NAMES])
    bad = np.flatnonzero(np.any(got != full, axis=0))
    assert bad.size == 0, ("delta arrays differ from a full transfer", bad[:10], stats.changed_count,
                           stats.full_transfer)
    for k in R.BUFFER_NAMES:
        assert np.array_equal(copy.arrays[k].view(np.uint32)[n:], before[k][n:]), "the tail beyond n was written"
    assert stats.surfel_count == n
    if n == 0 and expect != "fallback":   # nothing to select, nothing copied
        assert (stats.full_transfer, stats.changed_count, stats.d2h_bytes) == (0, 0, 0)
    elif expect == "fallback" or threshold <= 0:
        assert (stats.full_transfer, stats.changed_count, stats.d2h_bytes) == (1, n, 32 * n), (threshold, stats.changed_count)
        ledger.paths["fallback"] += 1
    else:
        new, window, merged = HW.delta_clauses(rows, token_count, token_epoch, threshold)
        changed = int((new | window | merged).sum())
        if 9 * changed > 8 * n:
            assert (stats.full_transfer, stats.changed_count, stats.d2h_bytes) == (1, n, 4 + 32 * n)
            ledger.paths["eight_ninths"] += 1
        else:
            assert stats.full_transfer == 0, (threshold, changed, n)
            assert stats.changed_count == changed, (stats.changed_count, changed, threshold)
            assert stats.d2h_bytes == 4 + 36 * changed
            ledger.paths["record"] += 1
            ledger.largest = max(ledger.largest, changed)
            ledger.merge_only += int((merged & ~new & ~window).sum())
    copy.ops = []
    return stats


def note(copies, frame, window):
    for c in copies:
        c.ops.append((frame, window))


def stream(stream_id=0, frames=24, cam=CAM):
    st = S.make_stream(cam, frames, stream_id=stream_id, device="cuda")
    others = R.stream_outlier_filter_transforms(st.global_T_frame, st.frame_T_global, K, st.depth_scaling)
    torch.cuda.synchronize()
    return st, others


def params(window):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = CAM.valid_region_radius()
    ip = IntegrateParams.defaults()
    ip.regularization_frame_window_size = window
    return pp, ip


def run_chunk(rec, st, others, pp, ip, first, last):
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, others, pp, ip, first, last)


class FrameIntegrator:
    """sm_preprocess + sm_integrate of one frame of a stream, at any frame index."""

    def __init__(self, rec, st, pp, ip):
        self.rec, self.st, self.pp, self.ip = rec, st, pp, ip
        H, W = CAM.height, CAM.width
        self.d = torch.zeros((H, W), dtype=torch.uint16, device="cuda")
        self.n = torch.zeros((H, W, 2), device="cuda")
        self.r = torch.zeros((H, W), device="cuda")

    def __call__(self, f, frame_index, window=None):
        st, ip = self.st, self.ip
        if window is not None:
            ip.regularization_frame_window_size = window
        others = [st.depth[o] for o in other_frames(f, self.pp.outlier_filtering_frame_count)]
        self.rec.preprocess(None, self.pp, st.depth[f], others, st.others_TR_reference[f], self.d, self.n, self.r)
        self.rec.integrate(None, frame_index, ip, self.d, self.n, self.r, st.color[f], st.global_T_frame[f],
                           st.frame_T_global[f])
        return ip.regularization_frame_window_size


@pytest.fixture(scope="module")
def streams():
    return stream(0), stream(3)


@pytest.fixture(scope="module")
def ledger():
    return Ledger()


@pytest.mark.parametrize("window", [5, 30])
def test_delta_after_stream_chunks(product, streams, ledger, window):
    (st, others), _ = streams
    pp, ip = params(window)
    rec = make(400_000)
    copy = Copy(400_000)
    first, last = st.integrated_range()
    delta(rec, copy, 0, ledger, expect="fallback")            # an empty cloud and a fresh token
    bounds = [first, first + 1, first + 3, first + 4, first + 7, first + 8, last]
    merge_only = ledger.merge_only
    for a, b in zip(bounds, bounds[1:]):
        run_chunk(rec, st, others, pp, ip, a, b)
        copy.ops += [(f, window) for f in range(a, b)]
        delta(rec, copy, b - 1, ledger)
    if window == 5:
        assert ledger.merge_only > merge_only, "no slot was selected by the merge clause alone"
    rec.close()


@pytest.mark.parametrize("window", [5, 30])
def test_delta_after_every_integrate(product, streams, ledger, window):
    (st, _), _ = streams
    pp, ip = params(window)
    rec = make(400_000)
    copy = Copy(400_000)
    integrate = FrameIntegrator(rec, st, pp, ip)
    first, last = st.integrated_range()
    merge_only = ledger.merge_only
    for f in range(first, last):
        integrate(f, 100 + f)
        note([copy], 100 + f, window)
        delta(rec, copy, 100 + f, ledger, expect="fallback" if f == first else None)
    if window == 5:     # at window 30 every stamp of this short stream stays inside the window
        assert ledger.merge_only > merge_only, "no slot was selected by the merge clause alone"
    rec.close()


def test_delta_after_every_session_push(product, streams, ledger):
    (st, _), _ = streams
    pp, ip = params(5)
    rec = make(400_000)
    copy = Copy(400_000)
    done = -1
    with rec.session(pp, ip, (CAM.width, CAM.height)) as s:
        for f in range(st.depth.shape[0]):
            status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            last = int(status.last_integrated_frame)
            copy.ops += [(g, 5) for g in range(done + 1, last + 1)]
            done = max(done, last)
            delta(rec, copy, max(last, 0), ledger, expect="fallback" if f == 0 else None)
    assert done > 10
    rec.close()


def test_delta_with_mixed_windows_and_two_tokens(product, streams, ledger):
    """Integrate() at window 30 and Regularize() at window 60 since a token: the smaller window start wins. Two copies
    filled in turn, as the reference's write / read double buffer does; a call with no operation since its token; a
    window reaching frame 0 falls back."""
    (st, _), _ = streams
    pp, ip = params(30)
    rec = make(400_000)
    a, b = Copy(400_000), Copy(400_000, pinned=True)
    integrate = FrameIntegrator(rec, st, pp, ip)
    first, last = st.integrated_range()
    base = 200
    for f in range(first, first + 3):
        integrate(f, base + f)
    delta(rec, a, base, ledger, expect="fallback")
    delta(rec, b, base, ledger, expect="fallback")
    for i, f in enumerate(range(first + 3, last)):
        integrate(f, base + f, 30)
        note([a, b], base + f, 30)
        rec.Regularize(None, base + f, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, 60)
        note([a, b], base + f, 60)
        delta(rec, (a, b)[i % 2], base + f, ledger)
    # nothing since the token: zero records, arrays bit-identical
    delta(rec, a, base + last, ledger)
    snapshot = {k: a.arrays[k].view(np.uint32).copy() for k in R.BUFFER_NAMES}
    stats = delta(rec, a, base + last, ledger)
    assert (stats.full_transfer, stats.changed_count, stats.d2h_bytes) == (0, 0, 4)
    for k in R.BUFFER_NAMES:
        assert np.array_equal(a.arrays[k].view(np.uint32), snapshot[k])
    # a window at or above the frame index: every stamp may have moved
    rec.Regularize(None, 50, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, 50)
    note([a, b], 50, 50)
    delta(rec, a, 50, ledger, expect="fallback")
    delta(rec, b, 50, ledger, expect="fallback")
    rec.close()


def test_delta_across_reset_and_load(product, streams, golden, ledger):
    (st, _), _ = streams
    pp, ip = params(5)
    rec = make(400_000)
    copy = Copy(400_000)
    integrate = FrameIntegrator(rec, st, pp, ip)
    first, last = st.integrated_range()
    for f in range(first, first + 3):
        integrate(f, 300 + f)
    delta(rec, copy, 300, ledger, expect="fallback")
    rec.reset()
    delta(rec, copy, 300, ledger, expect="fallback")          # n = 0 after the reset
    for f in range(first, first + 2):
        integrate(f, 300 + f)
        note([copy], 300 + f, 5)
    delta(rec, copy, 301, ledger)
    rows, merges = golden_state(golden, 7)
    rec.load_state(rows, merges)
    delta(rec, copy, 7, ledger, expect="fallback")
    rec.Regularize(None, 9, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, 3)
    note([copy], 9, 3)
    stats = delta(rec, copy, 9, ledger)
    assert stats.full_transfer == 0 and 0 < stats.changed_count < rows.shape[1]
    rec.close()


def test_delta_history_trim(product, golden, ledger):
    """More than 8192 operations since a token: the history keeps the newest 4097 after a trim. A token older than
    its front gets the full transfer; the one exactly one epoch before the front still takes the record path."""
    rows, merges = golden_state(golden, 7)
    n = rows.shape[1]
    rec = make(n + 64)
    rec.load_state(rows, merges)
    ip = IntegrateParams.defaults()
    copies = [Copy(n + 64) for _ in range(3)]
    for c in copies:
        delta(rec, c, 7, ledger, expect="fallback")
    frame = 100_000

    def regularize(count, window=10):
        for _ in range(count):
            rec.Regularize(None, frame, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, window)
            note(copies, frame, window)

    regularize(4095)
    delta(rec, copies[1], frame, ledger)            # epoch E0 + 4095: will be two before the front
    regularize(1)
    delta(rec, copies[2], frame, ledger)            # epoch E0 + 4096: will be one before the front
    regularize(8193 - 4096 - 1)
    regularize(1, window=frame - 6)                 # operation 8193: the trim; stamps >= 6 are in its window
    assert int(copies[2].token.epoch) == int(copies[0].token.epoch) + 4096
    s = delta(rec, copies[2], frame, ledger)
    assert s.full_transfer == 0 and s.changed_count == int((rows[18].view(np.int32) >= 6).sum()) > 0
    ledger.trim = (int(s.changed_count), int(copies[2].token.epoch))
    delta(rec, copies[1], frame, ledger, expect="fallback")
    delta(rec, copies[0], frame, ledger, expect="fallback")
    rec.close()


def test_delta_threaded_scatter_and_staging_growth(product, big, ledger):
    """On the state larger than one grid-stride pass: a window of about 10 k slots sizes the pinned staging at 2^20
    words; then about 150 k slots force it to grow and take the four-thread scatter; then a window of nearly every
    slot takes the 9/8 fallback."""
    rows, merges = big
    n = rows.shape[1]
    rec = make(n + 64)
    rec.load_state(rows, merges)
    ip = IntegrateParams.defaults()
    copy = Copy(n + 64, pinned=True)
    delta(rec, copy, 4000, ledger, expect="fallback")
    stamps = rows[18].view(np.int32)
    counts = []
    for target in (10_000, 150_000, int(0.95 * n)):
        window = 4000 - int(np.sort(stamps)[::-1][target])
        rec.Regularize(None, 4000, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, window)
        note([copy], 4000, window)
        s = delta(rec, copy, 4000, ledger)
        counts.append((int(s.changed_count), int(s.full_transfer)))
    (c1, f1), (c2, f2), (c3, f3) = counts
    assert f1 == 0 and 9 * c1 < (1 << 20)
    assert f2 == 0 and c2 >= 1 << 16 and 9 * c2 > 1 << 20 and 9 * c2 <= 8 * n
    assert f3 == 1 and c3 == n
    rec.close()


def test_delta_token_from_another_handle(product, streams, ledger):
    """A token and arrays filled from handle A, given to handle B that ran further (and to a handle created after A
    was destroyed): B's full transfer, never a delta against a cloud the arrays did not come from."""
    (st, others), (st2, others2) = streams
    pp, ip30 = params(30)
    _, ip5 = params(5)
    first, last = st.integrated_range()
    a = make(400_000)
    run_chunk(a, st2, others2, pp, ip30, first, first + 6)
    copy = Copy(400_000)
    delta(a, copy, first + 5, ledger, expect="fallback")
    b = make(400_000)
    run_chunk(b, st, others, pp, ip5, first, last)
    assert b.surfels_size() >= int(copy.token.surfel_count)
    delta(b, copy, last - 1, ledger, expect="fallback")
    b.close()
    a.close()
    # a token of a destroyed handle, on a handle created afterwards
    copy2 = Copy(400_000)
    a = make(400_000)
    run_chunk(a, st2, others2, pp, ip30, first, first + 4)
    delta(a, copy2, first + 3, ledger, expect="fallback")
    a.close()
    c = make(400_000)
    run_chunk(c, st, others, pp, ip5, first, last)
    delta(c, copy2, last - 1, ledger, expect="fallback")
    c.close()


def test_delta_reached_every_path(ledger):
    """Runs last in this module: the sequences above took the record path (the threaded scatter among them), both
    fallbacks, and the merge clause alone."""
    if not any(ledger.paths.values()):
        pytest.skip("only meaningful after the delta sequences of this module")
    print("\nhand-off delta: largest record count", ledger.largest, "merge-only selections", ledger.merge_only,
          "paths", ledger.paths, "trim", getattr(ledger, "trim", None))
    assert ledger.paths["record"] > 20 and ledger.paths["fallback"] > 5 and ledger.paths["eight_ninths"] >= 1
    assert ledger.largest >= 1 << 16 and ledger.merge_only > 0
