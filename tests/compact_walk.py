"""numpy restatement of sm_compact (include/surfel_b200.h, DESIGN.md section 5.13): the state a dump holds before
the call -> the state after it, the map and the stats."""
import numpy as np

INVALID = 0xFFFFFFFF
RADIUS_SQUARED_ROW = 7
LINK_ROWS = (19, 20, 21, 22)
SCRATCH_ROWS = (11, 12, 13, 14, 15, 16, 23)
CHECKED_ROWS = tuple(r for r in range(25) if r not in SCRATCH_ROWS)


def compact(rows, n, merge_count):
    """(rows [25, n] float32 of sm_dump_state, surfels_size, merge_count) -> (rows after, old_to_new uint32 [n],
    stats dict, merge_count after). Rule 1: a slot goes iff radius^2 < 0; rule 4: a merge count of 0, or no marked
    slot, changes nothing (identity map)."""
    rows = np.asarray(rows, np.float32)[:, :n]
    keep = ~(rows[RADIUS_SQUARED_ROW] < 0)
    identity = np.arange(n, dtype=np.uint32)
    unchanged = dict(slots_before=n, slots_after=n, merged_removed=0, links_dropped=0)
    if merge_count == 0 or n == 0 or keep.all():
        return rows.copy(), identity, unchanged, merge_count
    new = (np.cumsum(keep) - 1).astype(np.int64)
    old_to_new = np.where(keep, new, INVALID).astype(np.uint32)
    out = np.ascontiguousarray(rows[:, keep])
    dropped = 0
    for r in LINK_ROWS:
        v = out[r].view(np.uint32)
        named = v != INVALID
        to = np.full(v.shape, INVALID, np.uint32)
        inside = named & (v < n)
        to[inside] = old_to_new[v[inside].astype(np.int64)]
        dropped += int(np.count_nonzero(named & (to == INVALID)))
        out[r] = to.view(np.float32)
    kept = int(keep.sum())
    stats = dict(slots_before=n, slots_after=kept, merged_removed=n - kept, links_dropped=dropped)
    return out, old_to_new, stats, 0


def remap_triangles(triangles, old_to_new):
    """[T, 3] triangles over old slots -> over new slots, dropping a triangle with a removed corner."""
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    m = old_to_new.astype(np.int64)[t]
    return m[(m != INVALID).all(axis=1)].astype(np.uint32)
