"""sm_mesh_update on the GPU: after every update the full mesh equals sm_triangulate on the same handle and the
restatement (tests/mesh_walk.c) on sm_dump_state, bit for bit, and the added / removed lists are exactly the
differences from the previous update's mesh, in owner and umbrella order. Covers the host edit sequences, no
change, a whole new state, sm_reset, parameter changes, sm_triangulate in between, sessions in both modes,
sm_stream_run in two chunks, two handles, and the argument and capacity errors."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, MeshParams, MeshStats, MeshUpdateStats, PreprocessParams
from tests import mesh_update_walk as W
from tests import mesh_walk as M

pytestmark = pytest.mark.gpu

CAP = 2_000_000
STATS = [k for k, _ in MeshStats._fields_]


def make(cam, cap=CAP):
    return R.CUDASurfelReconstruction(cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


def loaded(rows, cap=None):
    rec = make(S.Camera.tum(320, 240), cap=cap or max(rows.shape[1] * 2, 1024))
    rec.load_state(rows, 0)
    return rec


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy().astype(np.uint32).reshape(-1, 3)


class Follower:
    """Updates one handle and checks every update against sm_triangulate, the walk and the previous mesh."""

    def __init__(self, rec, params=None):
        self.rec, self.params = rec, params
        self.previous = np.zeros((0, 3), np.uint32)
        self.deltas = []

    def update(self, walk=True):
        rec = self.rec
        st = rec.mesh_update(self.params)
        full, added, removed = (host(rec.mesh_triangles(w)) for w in ("all", "added", "removed"))
        ref, ref_stats = rec.triangulate(self.params)
        ref = host(ref)
        got = {k: int(getattr(st.mesh, k)) for k in STATS}
        assert got == {k: int(getattr(ref_stats, k)) for k in STATS}
        assert np.array_equal(full, ref), "full mesh differs from sm_triangulate"
        if walk:
            rows, _, _ = rec.dump_state()
            want, want_stats, _ = M.triangulate(rows, self.params)
            assert got == want_stats and np.array_equal(full, want), "full mesh differs from the restatement"
        prev = {tuple(t) for t in self.previous.tolist()}
        new = {tuple(t) for t in full.tolist()}
        assert st.triangles_added == len(added) and st.triangles_removed == len(removed)
        # exact lists: the set differences, in the order of the mesh they come from
        assert removed.tolist() == [t for t in self.previous.tolist() if tuple(t) not in new]
        assert added.tolist() == [t for t in full.tolist() if tuple(t) not in prev]
        rem, add = {tuple(t) for t in removed.tolist()}, {tuple(t) for t in added.tolist()}
        assert rem <= prev and not (add & (prev - rem)) and (prev - rem) | add == new
        self.previous = full
        self.deltas.append((added, removed))
        return st


def test_read_before_update_is_refused():
    rec = loaded(M.jittered_plane())
    count = C.c_uint64(7)
    buf = torch.zeros((10, 3), dtype=torch.int32, device="cuda")
    fn = rec.lib.fn["mesh_read"]
    for which in (0, 1, 2):
        assert fn(rec._h, None, which, C.c_void_p(buf.data_ptr()), 10, C.byref(count)) == _lib.SM_ERR_INVALID_ARGUMENT
    rec.close()


@pytest.mark.parametrize("name", ["jittered_plane", "pixel_grid", "sphere", "merged", "duplicates", "cube",
                                  "golden_f7"])
def test_edit_sequences(name):
    rows = M.golden_f7() if name == "golden_f7" else M.CASES[name]()
    steps = W.edit_sequence(rows, seed=7)
    rec = loaded(rows, cap=max(rows.shape[1] * 2, 1024))
    f = Follower(rec)
    first = f.update()
    assert first.full_sweep == 1 and first.triangles_removed == 0
    for label, new_rows in steps:
        rec.load_state(new_rows, 0)
        st = f.update()
        if label == "nudge_one_ulp" and name == "jittered_plane":
            assert st.slots_changed == 1 and 1 < st.umbrellas_rebuilt < 60 and st.full_sweep == 0
    rec.close()


@pytest.mark.parametrize("which", ["tie", "edge"])
def test_ties_and_ball_edges(which):
    rows, steps = W.tie_sequence() if which == "tie" else W.edge_sequence()
    rec = loaded(rows)
    f = Follower(rec)
    f.update()
    for _, new_rows in steps:
        rec.load_state(new_rows, 0)
        st = f.update()
        assert st.slots_changed == 1 and st.full_sweep == 0
    rec.close()


def test_no_change_and_triangulate_in_between():
    rows = M.golden_f7()
    rec = loaded(rows)
    f = Follower(rec)
    f.update()
    before = f.previous
    for _ in range(2):
        rec.triangulate(MeshParams(2.5, 40.0, 120.0))   # other params, its own buffers
        st = f.update()
        assert st.slots_changed == 0 and st.umbrellas_rebuilt == 0 and st.owners_rechecked == 0
        assert st.triangles_added == 0 and st.triangles_removed == 0
        assert np.array_equal(f.previous, before)
    rec.close()


def test_whole_new_state_reset_and_params():
    a = M.jittered_plane(seed=1)
    b = M.jittered_plane(seed=9)
    rec = loaded(a)
    f = Follower(rec)
    f.update()
    rec.load_state(b, 0)   # the same size, every slot moved
    st = f.update()
    assert st.full_sweep == 1 and st.slots_changed == a.shape[1]
    rec.reset()
    rec.load_state(b[:, :200], 0)   # smaller: everything is rebuilt
    st = f.update()
    assert st.full_sweep == 1 and st.owners_rechecked == a.shape[1]
    f.params = MeshParams(2.5, 40.0, 120.0)
    st = f.update()
    assert st.full_sweep == 1 and st.slots_changed == 0
    rec.reset()
    st = f.update()
    assert st.mesh.triangle_count == 0 and st.triangles_added == 0 and len(f.previous) == 0
    rec.close()


def test_errors_launch_nothing_and_capacity_writes_nothing():
    rec = loaded(M.jittered_plane())
    stats = MeshUpdateStats()
    fn = rec.lib.fn["mesh_update"]
    launches = rec.lib.fn["kernel_launch_count"]()
    for p in [MeshParams(0.0, 90, 170), MeshParams(math.nan, 90, 170), MeshParams(math.inf, 90, 170),
              MeshParams(2, 0.0, 170), MeshParams(2, 180.5, 170), MeshParams(2, 90, math.nan)]:
        assert fn(rec._h, None, C.byref(p), C.byref(stats)) == _lib.SM_ERR_INVALID_ARGUMENT
    assert rec.lib.fn["last_error"]() == b"sm_mesh_update: angles must be in (0, 180] degrees"
    p = MeshParams.defaults()
    assert fn(rec._h, None, None, C.byref(stats)) == _lib.SM_ERR_INVALID_ARGUMENT
    assert fn(rec._h, None, C.byref(p), None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert rec.lib.fn["kernel_launch_count"]() == launches
    want = rec.mesh_update().mesh.triangle_count
    read = rec.lib.fn["mesh_read"]
    count = C.c_uint64()
    buf = torch.full((want - 1, 3), -7, dtype=torch.int32, device="cuda")
    assert read(rec._h, None, 0, C.c_void_p(buf.data_ptr()), want - 1, C.byref(count)) == _lib.SM_ERR_CAPACITY
    assert rec.lib.fn["last_error"]() == f"sm_mesh_read: {want} triangles do not fit the capacity of {want - 1}".encode()
    torch.cuda.synchronize()
    assert count.value == want and (buf == -7).all()
    assert read(rec._h, None, 0, None, 0, C.byref(count)) == _lib.SM_ERR_CAPACITY and count.value == want
    assert read(rec._h, None, 3, C.c_void_p(buf.data_ptr()), want - 1, C.byref(count)) == _lib.SM_ERR_INVALID_ARGUMENT
    assert read(rec._h, None, 0, C.c_void_p(buf.data_ptr()), want - 1, None) == _lib.SM_ERR_INVALID_ARGUMENT
    rec.close()


@pytest.mark.parametrize("size,frames,serial", [((320, 240), 24, False), ((320, 240), 24, True),
                                                ((640, 480), 48, False), ((640, 480), 48, True)])
def test_sessions_update_after_every_push(size, frames, serial):
    cam = S.Camera.tum(*size)
    st = S.make_stream(cam, frames, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    rec = make(cam)
    if serial:
        rec.enable_timings(True)
    f = Follower(rec)
    sweeps = lists = 0
    with rec.session(pp, IntegrateParams.defaults(), (cam.width, cam.height)) as s:
        for k in range(st.frame_count):
            s.push(st.depth[k], st.color[k], st.global_T_frame[k], st.frame_T_global[k])
            u = f.update(walk=(k % 12 == 11))
            sweeps += u.full_sweep
            lists += 1 - u.full_sweep
    f.update()
    # (the regularisation window moves a large share of a cloud this young: most updates here are sweeps)
    print(f"{size} serial={serial}: {lists} list updates, {sweeps} sweeps")
    assert f.previous.shape[0] > 0
    rec.close()


def test_stream_run_in_two_chunks_and_two_handles():
    cam = S.Camera.tum(320, 240)
    st = S.make_stream(cam, 24, stream_id=3, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    first, last = st.integrated_range()
    mid = (first + last) // 2
    follow = []
    for _ in range(2):
        rec = make(cam)
        f = Follower(rec)
        for lo, hi in ((first, mid), (mid, last)):
            rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                           IntegrateParams.defaults(), lo, hi)
            f.update()
        follow.append(f.deltas)
        rec.close()
    for (a1, r1), (a2, r2) in zip(*follow):
        assert np.array_equal(a1, a2) and np.array_equal(r1, r2)


def test_sweep_taken_from_the_size_of_a():
    """Few slots change (|C| <= n / 16, so A is marked) but their balls reach more than 3/4 of the cloud: the
    umbrellas are rebuilt by the sweep inside the marked path, and the result is still exact."""
    params = MeshParams(3.0, 90.0, 170.0)
    rows = M.sphere()
    n = rows.shape[1]
    rec = loaded(rows)
    f = Follower(rec, params)
    f.update()
    pick = np.random.default_rng(3).choice(n, 120, replace=False)
    edited = rows.copy()
    edited[3, pick] = np.nextafter(edited[3, pick], np.float32(np.inf))
    rec.load_state(edited, 0)
    st = f.update()
    assert st.slots_changed == 120 and st.slots_changed * 16 <= n
    assert st.full_sweep == 1 and 4 * st.umbrellas_rebuilt > 3 * n and st.umbrellas_rebuilt < n
    rec.close()


def test_appended_slots_that_are_not_present():
    """Slots appended since the last update that are already merged own nothing and add nothing to the stats, also
    when the buffers grow for them and when a later update rebuilds everything."""
    rows = M.jittered_plane()
    n = rows.shape[1]
    rec = loaded(rows, cap=4 * n)
    f = Follower(rec)
    f.update()
    extra = np.concatenate([rows, rows], 1)
    extra[7, n:] = -1.0                                   # n merged slots: the per-slot buffers grow
    extra[7, n + 5] = rows[7, 5]                          # one of them present
    extra[3:6, n + 5] += np.float32(2e-3)
    rec.load_state(extra, 0)
    st = f.update()
    assert st.full_sweep == 0 and st.slots_changed == 1
    st = f.update()
    assert st.slots_changed == 0
    f.params = MeshParams(2.5, 90.0, 170.0)               # everything: every slot's share is recounted
    f.update()
    f.params = None
    f.update()
    rec.reset()
    rec.load_state(extra[:, : n + 10], 0)
    f.update()
    rec.close()
