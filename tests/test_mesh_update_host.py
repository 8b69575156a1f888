"""sm_mesh_update's rules checked on the CPU against the restatement (tests/mesh_update_walk.py over
tests/mesh_walk.c): on every edit of every hand-built cloud and the golden f7 state, the slots whose exact umbrella
changes are in A, the owners whose triangles or share of the stats change are in R, and the mesh assembled from
the previous mesh outside R and the new one inside R is the full mesh. Also the header's declaration of the calls."""
import re
from pathlib import Path

import numpy as np
import pytest

from tests import mesh_update_walk as W
from tests import mesh_walk as M

HEADER = Path(__file__).resolve().parents[1] / "include" / "surfel_b200.h"


def check_step(old, new, params=None, strict=False):
    """Asserts the three claims for one update old -> new; returns (C, A, R)."""
    a, c = W.rebuild_set(old.rows, new.rows, params, strict)
    r = W.recheck_set(old, a)
    for i in range(new.n):
        before = old.exact[i] if i < old.n else ()
        assert before == new.exact[i] or a[i], f"slot {i}: umbrella changed outside A"
    for o in range(max(old.n, new.n)):
        assert old.share(o) == new.share(o) or r[o], f"owner {o}: triangles or stats changed outside R"
    tri, stats = W.incremental(old, new, r)
    assert stats == new.stats
    assert np.array_equal(tri, new.tri)
    return c, a, r


def run_sequence(rows, steps):
    old = W.State(rows)
    out = []
    for label, new_rows in steps:
        new = W.State(new_rows)
        c, a, r = check_step(old, new)
        out.append((label, int(c.sum()), int(a.sum()), int(r.sum())))
        old = new
    return out


@pytest.mark.parametrize("name", sorted(M.CASES) + ["golden_f7"])
def test_rules_cover_every_edit(name):
    rows = M.golden_f7() if name == "golden_f7" else M.CASES[name]()
    sizes = run_sequence(rows, W.edit_sequence(rows, seed=7))
    assert sizes, name


def test_cocircular_tie_created_and_broken():
    rows, steps = W.tie_sequence()
    sizes = run_sequence(rows, steps)
    assert all(c == 1 for _, c, _, _ in sizes)


def test_neighbour_on_the_edge_of_a_ball():
    """A neighbour exactly on the edge of a ball counts (<=): with the strict variant of the test umbrellas change
    outside A (those slots then keep stale umbrellas), so this case tells the two apart."""
    rows, steps = W.edge_sequence()
    run_sequence(rows, steps)
    old = W.State(rows)
    missed = 0
    for _, new_rows in steps:
        new = W.State(new_rows)
        a, _ = W.rebuild_set(old.rows, new.rows, strict=True)
        missed += sum(1 for i in range(new.n) if old.exact[i] != new.exact[i] and not a[i])
        old = new
    assert missed > 0


def test_parameters_and_reset_rebuild_everything():
    """With other params, or a smaller cloud, the rules do not apply: the update rebuilds everything, which the
    assembly restates as R = every slot."""
    rows = M.jittered_plane()
    old = W.State(rows)
    new = W.State(rows[:, :300])
    tri, stats = W.incremental(old, new, np.ones(old.n, bool))
    assert stats == new.stats and np.array_equal(tri, new.tri)


def test_single_nudge_stays_local():
    rows = M.jittered_plane()
    label, nudged = W.edit_sequence(rows, seed=7)[0]
    assert label == "nudge_one_ulp"
    _, c, a, r = run_sequence(rows, [(label, nudged)])[0]
    assert c == 1 and 1 < a < 60 and a <= r < 120, (c, a, r)


def test_header_declares_the_calls():
    h = HEADER.read_text()
    assert "int sm_mesh_update(sm_reconstruction* r, void* stream, const sm_mesh_params* p, sm_mesh_update_stats* stats);" in h
    assert re.search(r"int sm_mesh_read\(sm_reconstruction\* r, void\* stream, int32_t which, uint32_t\* triangles", h)
    assert "sm_mesh_update, sm_mesh_read, sm_triangulate, sm_surfel_count" in h   # hand-off calls of a session
