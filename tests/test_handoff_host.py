"""The restatements of the hand-off (tests/handoff_walk.py) on hand-worked cases, and the constructed states they are
run on. No GPU needed."""
import numpy as np
import pytest

from tests import handoff_walk as HW
from tests.util import INVALID

GRAY = lambda v: int(HW.pack_rgb(v, v, v))


def test_stamp_threshold_is_the_smallest_window_start():
    assert HW.stamp_threshold([]) == HW.INT_MAX
    assert HW.stamp_threshold([(40, 30)]) == 10
    assert HW.stamp_threshold([(40, 30), (45, 60), (50, 5)]) == -15
    assert HW.stamp_threshold([(3, 5)]) == -2                    # the subtraction wraps in u32, then reads as int
    assert HW.stamp_threshold([(10, HW.INT_MAX)]) == 10 - HW.INT_MAX
    assert HW.stamp_threshold([(0, -5)]) == 5


@pytest.mark.parametrize("max_age", [1, 2, 30, HW.INT_MAX])
def test_age_ramp_by_hand(max_age):
    ages = np.array([-1, 0, 1, 2, max_age, max_age + 1] if max_age < HW.INT_MAX else [-1, 0, 1, 2, max_age])
    color, value = HW.age_ramp(ages, max_age)
    assert color[0] == color[1] == HW.RED                        # age < 1: updated in this frame (or later)
    assert color[2] == GRAY(255) and value[2] == 0               # age 1: the start of the ramp
    if max_age == 1:
        assert color[3] == HW.BLUE                               # beyond max_age (and 1 / 0 never evaluated)
        return
    want_2 = 0 if max_age == 2 else 255 - int(np.floor(HW.RAMP / (max_age - 1)))
    assert color[3] == GRAY(want_2)
    assert color[4] == GRAY(0) and value[4] == HW.RAMP           # blend 1: 255.99 truncates to 255
    if max_age < HW.INT_MAX:
        assert color[5] == HW.BLUE
    if max_age == 30:
        assert color[3] == GRAY(255 - 8)                         # 255.99 / 29 = 8.83


def test_age_below_the_stamp_wraps_to_a_negative_age():
    stamps = np.array([10, 5, 4, 0xFFFFFFF0], np.uint32)
    ages = HW.ages(stamps, 5)
    assert ages.tolist() == [-5, 0, 1, 21]
    color, _ = HW.age_ramp(ages, 30)
    assert color[0] == color[1] == HW.RED and color[2] == GRAY(255)


def test_flag_precedence_over_all_sixteen_combinations():
    for bits in range(16):
        last, creation, radii, normals = [(bits >> k) & 1 for k in range(4)]
        want = ("last_update" if last else "creation" if creation else "radii" if radii else
                "normals" if normals else "color")
        assert HW.viz_mode(last, creation, radii, normals) == want


def test_radius_ramp_by_hand():
    r2 = np.float32([-1.0, -0.0, 0.0, np.nan, 0.0005 ** 2, 0.01 ** 2, 1.0, 0.00525 ** 2])
    color, value = HW.radius_ramp(r2)
    red = (color & 0xFF).tolist()
    green = ((color >> 8) & 0xFF).tolist()
    assert red[:5] == [0, 0, 0, 0, 0]                             # sqrt(-1) and NaN saturate to 0, as does r < 0.5 mm
    assert red[5] in (254, 255) and red[6] == 255
    assert abs(value[7] - HW.RAMP * 0.5) < 1e-3 and red[7] == 127
    assert all(r + g == 255 for r, g in zip(red, green))
    assert np.all((color >> 16) == 80)


def test_normal_colors_by_hand():
    n = np.float32([[-1, 1, 0, 1.0001, -1.0001, np.float32(1) + np.float32(2.0 ** -23)],
                    [0, 0, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0]])
    color, value = HW.normal_colors(n)
    r = (color & 0xFF).tolist()
    assert r[0] == 0 and r[1] == 255 and r[2] == 127
    assert value[0, 3] > 256 and r[3] == 0                        # past 256 the u32 conversion's low byte wraps
    assert r[4] == 0                                             # negative: the conversion gives 0
    assert r[5] == 255                                           # one ulp above 1 stays below 256
    assert np.all(((color >> 8) & 0xFF) == 127)


def test_near_truncation():
    v = np.array([3.0, 3.00001, 2.99999, 3.5, np.nan, 3 + 2 * HW.NEAR])
    assert HW.near_truncation(v, HW.NEAR).tolist() == [True, True, True, False, False, False]


def _rows(n):
    rows = np.zeros((25, n), np.float32)
    rows[7] = 1e-4
    return rows


def test_vertex_buffer_gate_and_layout():
    rows = _rows(6)
    rows[3:6] = np.arange(18, dtype=np.float32).reshape(3, 6)
    rows[17] = np.uint32([4, 5, 6, 4, 5, 6]).view(np.float32)
    rows[24] = np.uint32([0x01ABCDEF] * 6).view(np.float32)
    out, close = HW.vertex_buffer(rows, 10, 30, 5, 3, "color")
    hidden = out[:, 0] == 0x7FFFFFFF
    # creation stamp after the last triangulation and a slot the mesh already has: x is NaN
    assert hidden.tolist() == [False, False, True, False, False, False]
    assert np.array_equal(out[:, 1:3], rows[4:6].view(np.uint32).T)
    assert np.all(out[:, 3] == 0x01ABCDEF) and not close.any()   # colour mode: the word as stored


def test_neighbor_segments_and_export():
    rows = _rows(3)
    rows[19:23] = np.uint32([[1, INVALID, 2], [INVALID, 0, 0], [2, 2, INVALID], [0, 1, 2]]).view(np.float32)
    seg = HW.neighbor_segments(rows)
    assert seg[0].tolist() == [0, 1, 0, 0, 0, 2, 0, 0]
    assert seg[1].tolist() == [1, 1, 1, 0, 1, 2, 1, 1]
    assert seg[2].tolist() == [2, 2, 2, 0, 2, 2, 2, 2]
    rows[7] = np.float32([-1, -0.0, np.nan])
    rows[3:6] = 7
    rows[24] = np.uint32([0x01020304, 0xFFAABBCC, 0]).view(np.float32)
    pos, col = HW.export_vertices(rows)
    assert np.all(pos[0] == 0x7FFFFFFF)                          # merged
    assert np.all(pos[1:].view(np.float32) == 7)                  # -0.0 and NaN are not below 0
    assert col.tolist() == [[4, 3, 2], [0xCC, 0xBB, 0xAA], [0, 0, 0]]


def test_delta_selection_clause_by_clause():
    n = 8
    rows = _rows(n)
    stamps = np.int64([5, 20, 19, 0, 0, 0, 30, 2 ** 31 + 5]).astype(np.uint32)
    rows[18] = stamps.view(np.float32)
    rows[7, [3, 4, 5]] = -1
    rows[14] = np.uint32([0, 0, 0, 7, 8, 9, 0, 0]).view(np.float32)
    # token: 7 slots, epoch 8; threshold 20
    new, window, merged = HW.delta_clauses(rows, 7, 8, 20)
    assert np.flatnonzero(new).tolist() == [7]
    assert np.flatnonzero(window).tolist() == [1, 6]              # stamp 2^31 + 5 reads as a negative int
    assert np.flatnonzero(merged).tolist() == [5]                 # merged at the token's epoch 8 (or 7): not since
    assert np.flatnonzero(HW.delta_selected(rows, 7, 8, 20)).tolist() == [1, 5, 6, 7]
    # each clause alone
    assert np.flatnonzero(HW.delta_selected(rows, 2, 9, HW.INT_MAX)).tolist() == [2, 3, 4, 5, 6, 7]
    assert np.flatnonzero(HW.delta_selected(rows, n, 9, 19)).tolist() == [1, 2, 6]
    assert np.flatnonzero(HW.delta_selected(rows, n, 6, HW.INT_MAX)).tolist() == [3, 4, 5]
    assert HW.delta_selected(rows, n, 9, HW.INT_MAX).sum() == 0
    # a threshold at or below 0 takes every stamp >= it, the merged slots' stamp 0 included
    assert np.flatnonzero(HW.delta_selected(rows, n, 9, 0)).tolist() == [0, 1, 2, 3, 4, 5, 6]


@pytest.mark.parametrize("n", [1, 33, 1000, 70_001])
def test_constructed_states_keep_the_invariants(n):
    rows, merges = HW.constructed_state(n)
    assert rows.shape == (25, n)
    assert merges == int((rows[7] < 0).sum())
    HW.check_constructed_invariants(rows)
    assert np.all(rows[18].view(np.uint32) < 2 ** 31)
    if n >= 70_000:
        r2 = rows[7]
        assert np.isnan(r2).any() and (r2 == -1).any() and (r2 == 0).any()
        assert (np.signbit(r2) & (r2 == 0)).any()                # -0.0
        assert np.isin(HW.radius_edges(), r2).all()              # every crossing of the radius ramp, +-64 ulps
        normals = rows[8:11]
        assert np.isin(HW.normal_edges(), normals).all()
        assert (np.abs(normals) > 1).any() and (normals == 1).any() and (normals == -1).any()
        assert (rows[19:23].view(np.uint32) == INVALID).any()
        _, value = HW.radius_ramp(r2)
        # the crossings are dense: hundreds of values within NEAR of a truncation point, on both sides
        assert HW.near_truncation(value, HW.NEAR).sum() > 1000
        stamps = rows[18].view(np.uint32)
        live = r2 >= 0
        assert stamps[live].min() <= 4000 - 3000 and stamps.max() >= 4001
