"""Regularize() against its float64 restatement (tests/reg_walk.py), at the resolution of the step.

The states are built to reach every branch of the sweeps: about 600 000 slots, several times the resident grid of
k_reg_accumulate and k_reg_step (4 blocks of 256 threads per SM), so that every thread runs the prefetch of a next
round; surfels on four planes with cut, invalid, self, duplicated and merged-slot links and one hub slot that about
200 slots link to; stamps that the window cuts; smooth positions up to 50 radii off on a subset, so that steps clamp.
Each sweep is held to the restatement's bound on every in-window slot, links and every other row bit-exact (except a
cut decision too close to call, and the slots that read it), slots outside the window bit-exact. Where the oracle is
built, the reference's kernels are held to the same restatement on the same states.
"""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200 import synthetic as S
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, SM_ERR_INVALID_ARGUMENT, SurfelError
from tests import reg_walk as W
from tests.util import NEIGHBOR_ROWS, SMOOTH_ROWS, check_state_invariants

pytestmark = pytest.mark.gpu

N = 600_000
GRID = 500                       # slots per row of a plane
SPACING = 0.004
FRAMES = (5, 1000, 2**31 - 2)
WINDOWS = (0, 3, 30, 2**30)
WEIGHTS = (0.0, 2.0, 10.0, 40.0, 1000.0)
RADIUS_FACTORS = (1.5, 2.0, 3.0)
HUB = N // 2 + 7 * GRID + 123
UNCHANGED_ROWS = [r for r in range(25) if r not in SMOOTH_ROWS + NEIGHBOR_ROWS + R.SCRATCH_ROWS]
CAM = (64, 48, 50.0, 50.0, 32.0, 24.0)


def constructed_state(frame_index, seed=7):
    """rows [25, N] and the merge count of a state with every kind of slot and link."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((25, N), np.float32)
    plane = np.arange(N) * 4 // N
    start = np.searchsorted(plane, np.arange(4))
    local = np.arange(N) - start[plane]
    uv = np.stack([local % GRID, local // GRID]).astype(np.float64) * SPACING
    normals = np.array([[0, 0, -1], [0.6, 0, -0.8], [0, 1, 0], [-0.48, 0.6, -0.64]], np.float64)
    origin = np.array([[0, 0, 2.0], [-1, 0.2, 1.5], [0.3, -0.8, 2.5], [2, -1, 3]], np.float64)
    a = np.cross(normals, [[1, 0, 0], [1, 0, 0], [0, 0, 1], [1, 0, 0]])
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    b = np.cross(normals, a)
    n = normals[plane].T + rng.normal(0, 0.02, (3, N))
    n = (n / np.linalg.norm(n, axis=0)).astype(np.float32)
    jitter = rng.normal(0, 0.1 * SPACING, (2, N))
    x = origin[plane].T + (uv[0] + jitter[0]) * a[plane].T + (uv[1] + jitter[1]) * b[plane].T
    x += normals[plane].T * rng.normal(0, 0.1 * SPACING, N)
    radius = SPACING * rng.uniform(0.7, 1.3, N)
    s = x + n * rng.normal(0, 0.2 * radius) + rng.normal(0, 0.05 * radius, (3, N))
    far = rng.random(N) < 0.03
    direction = rng.normal(size=(3, N))
    direction /= np.linalg.norm(direction, axis=0)
    s[:, far] = (x + direction * rng.uniform(0, 50, N) * radius)[:, far]
    rows[0:3], rows[3:6], rows[7], rows[8:11] = x, s, radius ** 2, n
    rows[6] = 1.0
    stamps = np.maximum(np.int64(frame_index) - rng.integers(0, 50, N), 0)
    stamps[rng.random(N) < 0.05] = frame_index
    stamps[HUB] = frame_index        # in every window: its 200 contributions always arrive
    color = rng.integers(0, 1 << 24, N).astype(np.uint32)
    merged = rng.random(N) < 0.01
    merged[HUB] = False
    rows[7, merged] *= -1
    stamps[merged] = 0
    detach = merged | (rng.random(N) < 0.005)
    color[detach] |= np.uint32(1 << 24)
    rows[17] = np.minimum(stamps, rng.integers(0, 50, N)).astype(np.uint32).view(np.float32)
    rows[18] = stamps.astype(np.uint32).view(np.float32)
    rows[24] = color.view(np.float32)
    # links: the four grid neighbours inside the plane, then replaced at random
    col, row = local % GRID, local // GRID
    rows_in_plane = np.bincount(plane, minlength=4)[plane]
    idx = np.arange(N, dtype=np.int64)
    links = np.stack([np.where(col > 0, idx - 1, idx + 1), np.where(col < GRID - 1, idx + 1, idx - 1),
                      np.where(row > 0, idx - GRID, idx + GRID),
                      np.where(local + GRID < rows_in_plane, idx + GRID, idx - GRID)])
    kind = rng.random((4, N))
    links = np.where(kind < 0.08, W.INVALID, links)
    links = np.where((kind >= 0.08) & (kind < 0.12), rng.integers(0, N, (4, N)), links)
    links = np.where((kind >= 0.12) & (kind < 0.14), idx, links)
    links[1:] = np.where((kind[1:] >= 0.14) & (kind[1:] < 0.17), links[0], links[1:])
    merged_slots = np.flatnonzero(merged)
    links = np.where((kind >= 0.17) & (kind < 0.20), merged_slots[rng.integers(0, len(merged_slots), (4, N))], links)
    # the hub: 200 slots around it link to it
    around = (HUB + GRID * np.arange(-10, 10)[:, None] + np.arange(-5, 5)[None, :]).ravel()
    links[3, around] = HUB
    rows[19:23] = links.astype(np.uint32).view(np.float32)
    return rows, int(merged.sum())


_STATES = {}


def state(frame_index):
    if frame_index not in _STATES:
        _STATES[frame_index] = constructed_state(frame_index)
    return _STATES[frame_index]


def make(lib=None):
    return R.CUDASurfelReconstruction(N, *CAM, lib=lib)


def check(rows, out, sweeps, label, excused=None):
    """Hold the dumped state `out` to the last of the restated `sweeps` run on `rows`. Returns the statistics.
    `excused`: bool mask of slots whose input smooth position or links the restatement does not know; they, the slots
    they link to or that link to them (in `rows` or in `out`), and what reads those in each sweep are not compared."""
    last = sweeps[-1]
    close = np.zeros(rows.shape[1], bool)
    for k, sweep in enumerate(sweeps):
        close = W.spread(close, sweep.links) if close.any() else close
        if k == 0 and excused is not None:
            for state in (rows, out):
                close |= W.spread(excused, state[list(NEIGHBOR_ROWS)].view(np.uint32))
        close |= sweep.cut_close.any(axis=0)
    links = out[list(NEIGHBOR_ROWS)].view(np.uint32)
    wrong_links = int(((links != last.links).any(axis=0) & ~close).sum())
    assert wrong_links == 0, f"{label}: {wrong_links} slots with links other than the restatement's"
    for r in UNCHANGED_ROWS:
        assert np.array_equal(out[r].view(np.uint32), rows[r].view(np.uint32)), f"{label}: row {r} changed"
    outside = ~np.logical_or.reduce([sw.inwin for sw in sweeps])
    if excused is not None:
        outside &= ~excused
    assert np.array_equal(out[3:6, outside].view(np.uint32), rows[3:6, outside].view(np.uint32)), \
        f"{label}: smooth positions outside the window moved"
    ratio = W.bound_ratio(out[3:6], last)
    checked = ~close
    worst = float(ratio[checked].max())
    bad = int((~(ratio <= 1.0) & checked).sum())
    assert bad == 0, f"{label}: {bad} slots beyond the bound (worst {worst:.3g} of it)"
    stats = dict(worst=worst, clamped=int(sum(sw.clamp.sum() for sw in sweeps)),
                 cut=int(sum(sw.cut.sum() for sw in sweeps)), outside=int(outside.sum()),
                 close=int(close.sum()), incoming=int(last.incoming.max()),
                 merged_in_window=int((last.inwin & (rows[7] < 0)).sum()),
                 detached=int(sum(sw.detached_links for sw in sweeps)))
    print(f"{label}: {stats}")
    return stats


def cases():
    """(frame, window, weight, radius factor): every frame index with every window, the weights and radius factors
    cycled through them, and all five weights at the default window."""
    out = []
    for i, (f, w) in enumerate([(f, w) for f in FRAMES for w in WINDOWS]):
        out.append((f, w, WEIGHTS[i % 5], RADIUS_FACTORS[i % 3]))
    out += [(1000, 30, weight, RADIUS_FACTORS[i % 3]) for i, weight in enumerate(WEIGHTS) if i != 2]
    return out


CASES = cases()


def run_cases(lib, label):
    rec = make(lib)
    totals = {}
    try:
        for frame_index, window, weight, rf in CASES:
            rows, merges = state(frame_index)
            rec.load_state(rows, merges)
            rec.Regularize(None, frame_index, weight, rf, window)
            out, n, _ = rec.dump_state()
            assert n == N
            sweep = W.regularize(rows, frame_index, window, weight, rf)
            stats = check(rows, out, [sweep], f"{label} frame {frame_index} window {window} w {weight} rf {rf}")
            assert stats["incoming"] >= 200, "the hub receives its contributions"
            for k, v in stats.items():
                totals[k] = max(totals.get(k, 0), v) if k == "worst" else totals.get(k, 0) + (v > 0)
    finally:
        rec.close()
    print(f"{label}: cases reaching each branch {totals}")
    assert totals["clamped"] > 0 and totals["cut"] > 0 and totals["outside"] > 0 and totals["merged_in_window"] > 0


def test_regularize_constructed_states(product):
    run_cases(None, "product")


def test_reference_kernels_constructed_states(reference):
    run_cases(reference, "reference")


def test_constructed_state_is_valid():
    rows, _ = state(FRAMES[0])
    check_state_invariants(rows, N)
    sweep = W.regularize(rows, 5, 30, 10.0, 2.0)
    assert sweep.incoming[HUB] >= 200


# ---------------------------------------------------------------------------------------------------------------
# the sweeps inside Integrate(): an all-invalid frame integrates nothing, so Integrate() is exactly its
# regularisation, with the detach pass over every slot that existed before the frame
# ---------------------------------------------------------------------------------------------------------------

def integrate_params(iterations, window=30, weight=10.0, rf=2.0):
    ip = IntegrateParams.defaults()
    ip.regularization_iterations_per_integration_iteration = iterations
    ip.regularization_frame_window_size = window
    ip.regularizer_weight = weight
    ip.radius_factor_for_regularization_neighbors = rf
    return ip


def expected_integrate(rows, frame_index, ip, remove_below=None, input_error=None):
    """The sweeps of Integrate()'s regularisation step on `rows`, the state the cycle left: the detach pass over the
    slots below `remove_below` (default: all; the slots that existed before the frame), and `input_error` [n] the
    euclidean bound of the input smooth positions (see "Chained sweeps" in reg_walk.py)."""
    window, weight, rf = (ip.regularization_frame_window_size, ip.regularizer_weight,
                          ip.radius_factor_for_regularization_neighbors)
    iterations = ip.regularization_iterations_per_integration_iteration
    if iterations == 0:
        return None
    remove_below = rows.shape[1] if remove_below is None else remove_below
    sweeps = [W.regularize(rows, frame_index, window, weight, rf, remove_below=remove_below, input_error=input_error)]
    for _ in range(1, iterations):
        prev = sweeps[-1]
        sweeps.append(W.regularize(rows, frame_index, window, weight, rf, smooth=prev.smooth, links=prev.links,
                                   input_error=np.sqrt(3) * prev.bound.max(axis=0)))
    return sweeps


def check_integrate(rows, out, frame_index, ip, label):
    sweeps = expected_integrate(rows, frame_index, ip)
    if sweeps is None:
        smooth, links = W.copy_only(rows, frame_index, ip.regularization_frame_window_size, remove_below=rows.shape[1])
        assert np.array_equal(out[3:6], smooth.astype(np.float32)), f"{label}: copy-only smooth positions"
        assert np.array_equal(out[list(NEIGHBOR_ROWS)].view(np.uint32), links), f"{label}: copy-only links"
        for r in UNCHANGED_ROWS:
            assert np.array_equal(out[r].view(np.uint32), rows[r].view(np.uint32)), f"{label}: row {r} changed"
        print(f"{label}: copy-only exact")
        return
    stats = check(rows, out, sweeps, label)
    assert stats["detached"] > 0


ITERATIONS = (0, 1, 2)


@pytest.mark.parametrize("iterations", ITERATIONS)
def test_integrate_empty_frame_regularizes(product, iterations):
    W_, H_ = CAM[0], CAM[1]
    frame_index = 1000
    rows, merges = state(frame_index)
    ip = integrate_params(iterations, window=3, weight=40.0, rf=1.5)
    rec = make()
    try:
        rec.load_state(rows, merges)
        zeros = torch.zeros((H_, W_), dtype=torch.uint16, device="cuda")
        rec.integrate(None, frame_index, ip, zeros, torch.zeros((H_, W_, 2), device="cuda"),
                      torch.zeros((H_, W_), device="cuda"), torch.zeros((H_, W_, 3), dtype=torch.uint8, device="cuda"),
                      np.eye(4, dtype=np.float32)[:3], np.eye(4, dtype=np.float32)[:3])
        out, n, m = rec.dump_state()
        assert (n, m) == (N, merges)
        check_integrate(rows, out, frame_index, ip, f"Integrate() iterations {iterations}")
    finally:
        rec.close()


@pytest.mark.parametrize("iterations", ITERATIONS)
def test_frame_graph_empty_frame_regularizes(product, iterations):
    """The same through sm_stream_run, which continues from the loaded state: one integrated all-zero frame."""
    W_, H_ = CAM[0], CAM[1]
    frame_index = 5
    rows, merges = state(frame_index)
    pp = PreprocessParams.defaults()
    K = pp.outlier_filtering_frame_count
    F = frame_index + K // 2 + 1
    ip = integrate_params(iterations, window=3, weight=10.0, rf=2.0)
    depth = torch.zeros((F, H_, W_), dtype=torch.uint16, device="cuda")
    color = torch.zeros((F, H_, W_, 3), dtype=torch.uint8, device="cuda")
    poses = np.tile(np.eye(4, dtype=np.float32)[:3], (F, 1, 1))
    others = np.tile(np.eye(4, dtype=np.float32)[:3], (F, K, 1, 1))
    rec = make()
    try:
        rec.load_state(rows, merges)
        stats = rec.stream_run(None, depth, color, poses, poses, others, pp, ip, frame_index, frame_index + 1)
        assert stats.frames_integrated == 1
        out, n, m = rec.dump_state()
        assert (n, m) == (N, merges)
        check_integrate(rows, out, frame_index, ip, f"frame graph iterations {iterations}")
    finally:
        rec.close()


# ---------------------------------------------------------------------------------------------------------------
# free-running handles: Regularize() on the state a stream left, with the record buffers and the previous sweep's
# threshold it carries, then once more straight after with a narrower window
# ---------------------------------------------------------------------------------------------------------------

def regularize_twice(rec, frame_index, ip, label):
    weight, rf = ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors
    window = ip.regularization_frame_window_size
    for step_window in (window, max(window // 2, 1)):
        rows, n, _ = rec.dump_state()
        rec.Regularize(None, frame_index, weight, rf, step_window)
        out = rec.dump_state()[0]
        check(rows, out, [W.regularize(rows, frame_index, step_window, weight, rf)],
              f"{label} window {step_window} (n {n})")


@pytest.mark.parametrize("window", [3, None])
def test_free_running_stream_handle(product, window):
    cam = S.Camera.tum(320, 240)
    st = S.make_stream(cam, 24, stream_id=21, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    if window is not None:
        ip.regularization_frame_window_size = window
    first, last = st.integrated_range()
    rec = R.CUDASurfelReconstruction(400_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    try:
        rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                       first, last)
        regularize_twice(rec, last - 1, ip, f"stream_run window {ip.regularization_frame_window_size}")
    finally:
        rec.close()


def test_free_running_session_handle(product):
    cam = S.Camera.tum(320, 240)
    st = S.make_stream(cam, 24, stream_id=21, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    ip.regularization_frame_window_size = 4
    rec = R.CUDASurfelReconstruction(400_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    done = []
    try:
        with rec.session(pp, ip, (cam.width, cam.height)) as s:
            for f in range(st.depth.shape[0]):
                status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
                if status.last_integrated_frame == 12 and not done:
                    regularize_twice(rec, 12, ip, "session")
                    done.append(12)
        assert done
    finally:
        rec.close()


# ---------------------------------------------------------------------------------------------------------------
# frame indices from 2^31 up are refused
# ---------------------------------------------------------------------------------------------------------------

def test_frame_indices_from_2_31_are_refused(product):
    rows, merges = state(FRAMES[-1])
    rec = make()
    try:
        rec.load_state(rows, merges)
        before = rec.dump_state()[0]
        with pytest.raises(SurfelError) as e:
            rec.Regularize(None, 2**31, 10.0, 2.0, 30)
        assert e.value.code == SM_ERR_INVALID_ARGUMENT
        W_, H_ = CAM[0], CAM[1]
        zeros = torch.zeros((H_, W_), dtype=torch.uint16, device="cuda")
        with pytest.raises(SurfelError) as e:
            rec.integrate(None, 2**32 - 1, IntegrateParams.defaults(), zeros, torch.zeros((H_, W_, 2), device="cuda"),
                          torch.zeros((H_, W_), device="cuda"),
                          torch.zeros((H_, W_, 3), dtype=torch.uint8, device="cuda"),
                          np.eye(4, dtype=np.float32)[:3], np.eye(4, dtype=np.float32)[:3])
        assert e.value.code == SM_ERR_INVALID_ARGUMENT
        assert np.array_equal(rec.dump_state()[0].view(np.uint32), before.view(np.uint32)), "nothing was launched"
        high = rows.copy()
        high[18, 17] = np.uint32(2**31).view(np.float32)
        with pytest.raises(SurfelError) as e:
            rec.load_state(high, merges)
        assert e.value.code == SM_ERR_INVALID_ARGUMENT
        assert np.array_equal(rec.dump_state()[0].view(np.uint32), before.view(np.uint32)), "the state is kept"
        # the largest frame index still accepted
        rec.Regularize(None, 2**31 - 1, 10.0, 2.0, 30)
    finally:
        rec.close()
