"""The float64 restatement of Regularize() (tests/reg_walk.py) against the reference's recorded answer and against
hand-built states with closed-form answers."""
import numpy as np
import pytest

from tests import reg_walk as W
from tests.util import GOLDEN_DIR, INTEGRATE_ROWS, NEIGHBOR_ROWS, digest, load_npz_xz, oracle_answers

INV = W.INVALID


def test_restatement_matches_reference_on_golden_state(golden):
    """Regularize() with the default settings on the reference's state after the golden frames: every slot, merged
    ones included, within the bound of the reference's own answer, and its links (and every row the call must not
    change) equal to the recorded digests."""
    last = int(golden["frames"][1])
    rows = golden[f"f{last - 1}_state"]
    assert digest(rows) == oracle_answers()["golden_handoff"]["inputs"]
    sweep = W.regularize(rows, last, 30, 10.0, 2.0)
    smooth_r = load_npz_xz(GOLDEN_DIR / "oracle_regularized_smooth.npz.xz")["smooth"]
    ratio = W.bound_ratio(smooth_r, sweep)
    assert np.isfinite(ratio).all() and ratio.max() <= 1.0, f"worst slot uses {ratio.max():.3f} of its bound"
    merged = rows[7] < 0
    assert merged.any() and sweep.inwin[merged].all(), "merged slots are part of this case"
    # the bound resolves the step: a step off by 1 % leaves it on most moving slots
    step = np.abs(sweep.smooth - rows[3:6]).max(axis=0)
    moving = step > 0
    assert np.median(sweep.bound.max(axis=0)[moving] / step[moving]) < 1e-2
    out = rows.copy()
    out[list(NEIGHBOR_ROWS)] = sweep.links.view(np.float32)
    answers = oracle_answers()["golden_handoff"]["regularized_rows"]
    assert {str(r): digest(out[r].view(np.uint32)) for r in INTEGRATE_ROWS + NEIGHBOR_ROWS} == answers


def state(x, s, normals, r2, stamps, links, detach=None):
    """rows [25, n] of a hand-built state."""
    n = len(x)
    rows = np.zeros((25, n), np.float32)
    rows[0:3] = np.asarray(x, np.float32).T
    rows[3:6] = np.asarray(s, np.float32).T
    rows[7] = r2
    rows[8:11] = np.asarray(normals, np.float32).T
    rows[18] = np.asarray(stamps, np.uint32).view(np.float32)
    rows[19:23] = np.asarray(links, np.uint32).T.copy().view(np.float32)
    color = np.full(n, 0x00808080, np.uint32)
    if detach is not None:
        color[np.asarray(detach)] |= np.uint32(1 << 24)
    rows[24] = color.view(np.float32)
    return rows


Z = (0.0, 0.0, 1.0)


def f64(rows, r):
    return rows[r].astype(np.float64)


def test_coplanar_neighbours_add_nothing():
    """Neighbours in the slot's tangent plane: only the data term and the weight sum act."""
    w = 10.0
    x = [(0, 0, 1), (0.004, 0, 1), (0, 0.004, 1)]
    s = [(0.001, 0.0005, 1), (0.004, 0, 1), (0, 0.004, 1)]
    rows = state(x, s, [Z] * 3, 1e-4, [5] * 3, [(1, 2, INV, INV), (0, INV, INV, INV), (0, INV, INV, INV)])
    sweep = W.regularize(rows, 5, 30, w, 2.0)
    # slot 0 receives w / 1 from slots 1 and 2
    expected = f64(rows, slice(3, 6))[:, 0] - (f64(rows, slice(3, 6))[:, 0] - f64(rows, slice(0, 3))[:, 0]) / (1 + w + 2 * w)
    assert np.allclose(sweep.smooth[:, 0], expected, rtol=0, atol=1e-15)
    assert np.array_equal(sweep.smooth[:, 1:], f64(rows, slice(3, 6))[:, 1:])
    assert list(sweep.incoming) == [2, 1, 1]


@pytest.mark.parametrize("w", [0.5, 10.0, 1000.0])
def test_two_surfel_pair(w):
    """Two slots linked to each other, parallel normals, 2 mm apart along them: both terms pull them together."""
    h = np.float32(0.002)
    rows = state([(0, 0, 0), (0.01, 0, h)], [(0, 0, 0), (0.01, 0, h)], [Z, Z], 0.01, [3, 3],
                 [(1, INV, INV, INV), (0, INV, INV, INV)])
    sweep = W.regularize(rows, 3, 30, w, 2.0)
    move = 2 * w * float(h) / (1 + 2 * w)     # slot 0: acc = nb = -2 w h along z, sf = 0.5 / (1 + 2w)
    assert np.allclose(sweep.smooth[2], [move, float(h) - move], rtol=1e-14, atol=0)
    assert np.array_equal(sweep.smooth[:2], f64(rows, slice(3, 5)))
    assert not sweep.clamp.any() and not sweep.cut.any()


def test_clamped_step_has_the_length_of_the_radius():
    r = 0.001
    rows = state([(0, 0, 2)], [(0.3, -0.4, 2.0)], [Z], r * r, [4], [(INV,) * 4])
    sweep = W.regularize(rows, 4, 30, 10.0, 2.0)
    assert sweep.clamp.all()
    step = f64(rows, slice(3, 6))[:, 0] - sweep.smooth[:, 0]
    assert np.isclose(np.linalg.norm(step), float(np.sqrt(np.float32(r * r))), rtol=1e-14)
    assert np.allclose(step / np.linalg.norm(step), [0.6, -0.8, 0], atol=1e-7)


def test_merged_slot_never_clamps():
    rows = state([(0, 0, 2)], [(0.3, -0.4, 2.0)], [Z], -1e-6, [0], [(INV,) * 4])
    sweep = W.regularize(rows, 4, 30, 10.0, 2.0)
    assert not sweep.clamp.any()
    assert np.allclose(sweep.smooth[:, 0], f64(rows, slice(0, 3))[:, 0] + (f64(rows, slice(3, 6))[:, 0] - f64(rows, slice(0, 3))[:, 0]) * (1 - 1 / 11))


def test_self_link_and_duplicated_link():
    """Slot 0 links itself once and slot 1 twice: count 3, the self term is zero but takes its share of the weight;
    slot 1 gets two contributions."""
    w, h = 6.0, float(np.float32(0.003))
    rows = state([(0, 0, 0), (0.002, 0, h)], [(0, 0, 0), (0.002, 0, h)], [Z, Z], 0.01, [2, 2],
                 [(0, 1, 1, INV), (INV,) * 4])
    sweep = W.regularize(rows, 2, 30, w, 2.0)
    assert list(sweep.incoming) == [1, 2]
    # slot 0: acc 0, wsum w/3; nb = (2w/3) * (2 h) along -z (two links to slot 1, the self term 0)
    g0 = -(2 * w / 3) * 2 * h
    assert np.isclose(sweep.smooth[2, 0], -0.5 / (1 + w + w / 3) * g0, rtol=1e-14)
    # slot 1: acc = 2 * (2w/3) * n.(s_1 - s_0) = 2 * (2w/3) * h along z, wsum 2w/3, no links of its own
    g1 = 2 * (2 * w / 3) * h
    assert np.isclose(sweep.smooth[2, 1], h - 0.5 / (1 + w + 2 * w / 3) * g1, rtol=1e-14)


def test_far_link_is_cut_only_when_used():
    """A link longer than rf * radius is cut when the neighbour is in the window, kept when it is not."""
    rows = state([(0, 0, 0), (1, 0, 0), (0, 1, 0)], [(0, 0, 0), (1, 0, 0), (0, 1, 0)], [Z] * 3, 1e-4, [9, 9, 1],
                 [(1, 2, INV, INV), (INV,) * 4, (INV,) * 4])
    sweep = W.regularize(rows, 9, 3, 10.0, 2.0)
    assert list(sweep.links[:, 0]) == [INV, 2, INV, INV]
    assert sweep.cut[0, 0] and not sweep.cut[1, 0]
    assert not sweep.inwin[2] and sweep.smooth[0, 2] == 0.0


def test_link_to_detached_slot():
    """The detach pass drops links to slots with colour byte 3 = 1, only for slots below remove_below."""
    x = [(0, 0, 0), (0.001, 0, 0), (0, 0.001, 0)]
    links = [(1, 2, INV, INV), (0, 2, INV, INV), (INV,) * 4]
    rows = state(x, x, [Z] * 3, 1e-4, [5] * 3, links, detach=[2])
    sweep = W.regularize(rows, 5, 30, 10.0, 2.0, remove_below=1)
    assert list(sweep.links[:, 0]) == [1, INV, INV, INV] and list(sweep.links[:, 1]) == [0, 2, INV, INV]
    assert sweep.detached_links == 1 and list(sweep.incoming) == [1, 1, 1]
    smooth, copied = W.copy_only(rows, 5, 30, remove_below=3)
    assert list(copied[:, 1]) == [0, INV, INV, INV]
    assert np.array_equal(smooth, f64(rows, slice(0, 3)))


def test_frame_index_below_window():
    """frame_index - window wraps below zero: the threshold is negative and every slot, stamp 0 included, moves."""
    assert W.threshold(2, 30) == -28
    x = [(0, 0, 1), (0.001, 0, 1)]
    s = [(0, 0, 1.0005), (0.001, 0, 1.0005)]
    rows = state(x, s, [Z, Z], 1e-4, [0, 2], [(1, INV, INV, INV), (0, INV, INV, INV)])
    sweep = W.regularize(rows, 2, 30, 10.0, 2.0)
    assert sweep.inwin.all()
    assert (sweep.smooth[2] != f64(rows, 5)).all()


def test_window_zero():
    """Window 0: only slots stamped with this frame index move or receive contributions; the others keep their smooth
    position exactly, and their links still give to in-window slots."""
    x = [(0, 0, 1), (0.001, 0, 1), (0, 0.001, 1)]
    s = [(0, 0, 1.0005), (0.001, 0, 1.001), (0, 0.001, 1.0002)]
    rows = state(x, s, [Z] * 3, 1e-4, [7, 6, 7], [(1, 2, INV, INV), (0, INV, INV, INV), (0, INV, INV, INV)])
    sweep = W.regularize(rows, 7, 0, 10.0, 2.0)
    assert list(sweep.inwin) == [True, False, True]
    assert np.array_equal(sweep.smooth[:, 1], f64(rows, slice(3, 6))[:, 1]) and sweep.bound[:, 1].max() == 0
    assert list(sweep.incoming) == [2, 0, 1]   # slot 0 uses only slot 2; slot 1, outside, still gives to 0
    _, copied = W.copy_only(rows, 7, 0)
    assert np.array_equal(copied, rows[19:23].view(np.uint32))


def test_weight_zero_returns_the_measurement():
    """w = 0: s' = s - (s - x) = x unless the step is clamped; far links are still cut."""
    x = [(0, 0, 1), (0.5, 0, 1)]
    s = [(0, 0.0001, 1.0002), (0.5, 0, 1.0001)]
    rows = state(x, s, [Z, Z], 1e-4, [3, 3], [(1, INV, INV, INV), (INV,) * 4])
    sweep = W.regularize(rows, 3, 30, 0.0, 2.0)
    assert np.allclose(sweep.smooth, f64(rows, slice(0, 3)), rtol=0, atol=1e-16)
    assert sweep.cut[0, 0]


def test_bound_compounds_through_chained_sweeps():
    """An input error grows by at most 1 + 2 sf dg / Delta per sweep, i.e. under 5-fold."""
    rng = np.random.default_rng(3)
    n = 200
    x = np.c_[rng.uniform(0, 0.05, n), rng.uniform(0, 0.05, n), np.full(n, 1.0)]
    s = x + rng.normal(0, 2e-4, (n, 3))
    links = rng.integers(0, n, (n, 4)).astype(np.uint32)
    rows = state(x, s, [Z] * n, 4e-4, [5] * n, links)
    first = W.regularize(rows, 5, 30, 10.0, 3.0)
    delta = np.full(n, 1e-6)
    second = W.regularize(rows, 5, 30, 10.0, 3.0, smooth=first.smooth, links=first.links, input_error=delta)
    own = W.regularize(rows, 5, 30, 10.0, 3.0, smooth=first.smooth, links=first.links)
    carried = second.bound - own.bound
    assert (carried >= delta - 1e-18).all() and (carried <= 5 * delta).all()
