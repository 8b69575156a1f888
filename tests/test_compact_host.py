"""sm_compact's numpy restatement (tests/compact_walk.py) on hand-worked cases and on the golden states."""
import numpy as np
import pytest

from tests import compact_walk as W
from tests.util import load_golden

INV = W.INVALID


def state(n, merged=(), links=None):
    """A hand-built state: row r of slot i = 1000 r + i, radius^2 -1 for the merged slots, and links[i] (up to 4
    slot numbers) in rows 19-22 (INV where not given)."""
    rows = (np.arange(25, dtype=np.float32)[:, None] * 1000 + np.arange(n, dtype=np.float32)[None]).astype(np.float32)
    rows[7] = 0.01
    rows[7, list(merged)] = -1.0
    link = np.full((4, n), INV, np.uint32)
    for i, named in (links or {}).items():
        link[:len(named), i] = named
    rows[19:23] = link.view(np.float32)
    return rows


def links(rows):
    return rows[19:23].view(np.uint32)


def test_none_merged_is_the_identity():
    rows = state(5)
    out, m, stats, merges = W.compact(rows, 5, 0)
    assert np.array_equal(out.view(np.uint32), rows.view(np.uint32))
    assert m.tolist() == [0, 1, 2, 3, 4] and stats["merged_removed"] == 0 and merges == 0


def test_merge_count_without_marks_changes_nothing():
    rows = state(4)
    out, m, stats, merges = W.compact(rows, 4, 3)
    assert np.array_equal(out.view(np.uint32), rows.view(np.uint32)) and merges == 3
    assert m.tolist() == [0, 1, 2, 3] and stats["slots_after"] == 4


def test_all_merged():
    rows = state(6, merged=range(6), links={0: [1, 2]})
    out, m, stats, merges = W.compact(rows, 6, 6)
    assert out.shape == (25, 0) and (m == INV).all() and merges == 0
    assert stats == dict(slots_before=6, slots_after=0, merged_removed=6, links_dropped=0)


def test_alternating():
    rows = state(8, merged=range(1, 8, 2), links={0: [1, 2, 4], 2: [0, 3], 6: [INV, 7, 6]})
    out, m, stats, _ = W.compact(rows, 8, 4)
    assert m.tolist() == [0, INV, 1, INV, 2, INV, 3, INV]
    assert out[0].tolist() == [0, 2, 4, 6] and out[24].tolist() == [24000, 24002, 24004, 24006]
    assert links(out)[:, 0].tolist() == [INV, 1, 2, INV]        # 1 removed, 2 -> 1, 4 -> 2
    assert links(out)[:, 1].tolist() == [0, INV, INV, INV]      # 3 removed
    assert links(out)[:, 3].tolist() == [INV, INV, 3, INV]      # an invalid link stays, 7 removed, 6 -> 3
    assert stats["links_dropped"] == 3                          # 1, 3, 7: the invalid link is not counted


def test_segment_boundary_and_end():
    n = 2050
    rows = state(n, merged=[1023, 1024, n - 1], links={1025: [1022, 1023, 1024, 1026], 0: [n - 1, n - 2]})
    out, m, stats, _ = W.compact(rows, n, 3)
    assert m[1022] == 1022 and m[1023] == INV and m[1024] == INV and m[1025] == 1023 and m[n - 1] == INV
    assert m[n - 2] == n - 4 and stats["slots_after"] == n - 3
    assert links(out)[:, 1023].tolist() == [1022, INV, INV, 1024]
    assert links(out)[:, 0].tolist() == [INV, n - 4, INV, INV]
    assert stats["links_dropped"] == 3


def test_merged_slot_linking_to_itself_and_links_beyond_n():
    rows = state(4, merged=[2], links={2: [2], 1: [2, 9]})
    out, m, stats, _ = W.compact(rows, 4, 1)
    assert out.shape[1] == 3 and links(out)[:, 1].tolist() == [INV, INV, INV, INV]
    assert stats["links_dropped"] == 2   # a kept slot's link to the removed slot, and one past surfels_size()


def test_nan_and_negative_zero_radius_are_kept():
    rows = state(3, merged=[0])
    rows[7, 1] = np.float32(-0.0)
    rows[7, 2] = np.nan
    _, m, stats, _ = W.compact(rows, 3, 1)
    assert m.tolist() == [INV, 0, 1] and stats["merged_removed"] == 1


def test_remap_triangles_drops_removed_corners():
    m = np.array([0, INV, 1, 2], np.uint32)
    assert W.remap_triangles([[0, 2, 3], [0, 1, 2]], m).tolist() == [[0, 1, 2]]


@pytest.mark.parametrize("frame", [4, 5, 6, 7])
def test_golden_states_keep_their_live_slots_in_order(frame):
    g = load_golden()
    rows = g[f"f{frame}_state"]
    n = rows.shape[1]
    live = ~(rows[7] < 0)
    out, m, stats, merges = W.compact(rows, n, int(g[f"f{frame}_counts"][1]))
    if stats["merged_removed"] == 0:
        assert merges == int(g[f"f{frame}_counts"][1])
        return
    assert stats["slots_after"] == int(live.sum()) and merges == 0
    assert np.array_equal(out[0].view(np.uint32), rows[0, live].view(np.uint32))
    kept = m[live].astype(np.int64)
    assert np.array_equal(kept, np.arange(kept.size))
    assert (links(out) == INV).sum() >= (rows[19:23, live].view(np.uint32) == INV).sum()
