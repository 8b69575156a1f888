"""The keyframe database and sm_relocalise on the GPU: codes, distances, query order and add decisions bit for bit
against the numpy restatement (tests/reloc_walk.py), determinism, relocalisation against sm_track_frame /
sm_track_frame_rgbd, read-only behaviour, launch counts and argument checks, kidnapped cameras, and pose-free
sessions that lose the camera and get it back."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import PreprocessParams, RelocParams, RelocResult, TrackRGBDParams
from tests import reloc_walk as W
from tests import track_walk as TW
from tests.util import offset, params

pytestmark = pytest.mark.gpu

VGA = S.Camera.tum(640, 480)
SMALL = S.Camera.tum(160, 120)
CAP = 2_000_000
MAX_T, MAX_R = 0.01, 0.5   # test_track_gpu.py::test_pose_free_stream at nominal noise


def make(cam=VGA):
    return R.CUDASurfelReconstruction(CAP, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


def with_(base=None, **kw):
    p = RelocParams.defaults() if base is None else RelocParams.from_buffer_copy(base)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def odd_camera():
    return S.Camera(331, 247, 271.5, 271.5, 165.3, 123.9)


@pytest.mark.parametrize("cam", [VGA, S.Camera.tum(320, 240), odd_camera()], ids=["640x480", "320x240", "331x247"])
def test_encode_is_exact_against_the_restatement(cam):
    st = S.make_stream(cam, 3, device="cuda")
    rec = make(cam)
    checked = 0
    for level in (1, 2, 3, 4):
        w, h = W.fern_size(cam.width, level), W.fern_size(cam.height, level)
        fits = -(-cam.width // w) <= 16 and -(-cam.height // h) <= 16
        for ferns in ((8, 512, 2048) if level == 3 else (512,)):
            p = with_(level=level, ferns=ferns, seed=1000 + level)
            if not fits:
                with pytest.raises(_lib.SurfelError):
                    R.KeyframeDatabase(rec, p)
                continue
            db = R.KeyframeDatabase(rec, p)
            enc = W.Encoder.of(cam.width, cam.height, p)
            for f in range(st.frame_count):
                got = db.encode(st.depth[f], st.color[f]).cpu().numpy().view(np.uint32)
                want = enc.encode(st.depth[f].cpu().numpy(), st.color[f].cpu().numpy())
                assert np.array_equal(got, want), (level, ferns, f)
                checked += 1
            db.close()
    assert checked >= 9


@pytest.fixture(scope="module")
def small_stream():
    return S.make_stream(SMALL, 240, device="cuda")


def test_query_distances_and_order_are_exact(small_stream):
    st = small_stream
    rec = make(SMALL)
    p = with_(candidates=8, max_query_fraction=1.0, capacity=600)
    db = R.KeyframeDatabase(rec, p)
    enc = W.Encoder.of(SMALL.width, SMALL.height, p)
    codes = []
    for f in range(st.frame_count):
        for _ in range(2 if f % 3 == 0 else 1):   # every third frame twice: equal distances
            index, full = db.add(st.depth[f], st.color[f], st.global_T_frame[f], force=True)
            assert index == len(codes) and not full
            codes.append(enc.encode(st.depth[f].cpu().numpy(), st.color[f].cpu().numpy()))
    assert len(db) == len(codes) > 300
    for i in (0, 1, 17, len(codes) - 1):
        assert np.array_equal(db.code(i), codes[i])
    for f in (0, 3, 50, 121, 239):
        idx, dist = db.query(st.depth[f], st.color[f])
        q = enc.encode(st.depth[f].cpu().numpy(), st.color[f].cpu().numpy())
        want_i, want_d = W.query(q, codes, 8, 1.0, p.ferns)
        assert idx.tolist() == want_i.tolist() and dist.tolist() == want_d.tolist(), f
        assert dist[0] == 0 and (f % 3 != 0 or dist[1] == 0)   # the frame itself (twice when it was stored twice)
    # a tight bound drops the far candidates
    tight = with_(p, max_query_fraction=0.05)
    dbt = R.KeyframeDatabase(rec, tight)
    for f in range(0, st.frame_count, 7):
        dbt.add(st.depth[f], st.color[f], st.global_T_frame[f], force=True)
    stored = [codes[sum(2 if g % 3 == 0 else 1 for g in range(f))] for f in range(0, st.frame_count, 7)]
    idx, dist = dbt.query(st.depth[100], st.color[100])
    q = enc.encode(st.depth[100].cpu().numpy(), st.color[100].cpu().numpy())
    want_i, want_d = W.query(q, stored, tight.candidates, 0.05, p.ferns)
    assert idx.tolist() == want_i.tolist() and dist.tolist() == want_d.tolist()


def run_adds(st, p, rec):
    db = R.KeyframeDatabase(rec, p)
    out = [db.add(st.depth[f], st.color[f], st.global_T_frame[f], force=(f % 50 == 49)) for f in range(st.frame_count)]
    return db, out


def test_add_decisions_are_exact_over_a_stream(small_stream):
    st = small_stream
    rec = make(SMALL)
    p = with_(capacity=12, add_fraction=0.05)
    db, got = run_adds(st, p, rec)
    enc = W.Encoder.of(SMALL.width, SMALL.height, p)
    ref = W.Database(p.ferns, p.capacity, p.add_fraction)
    want = [ref.add(enc.encode(st.depth[f].cpu().numpy(), st.color[f].cpu().numpy()), st.global_T_frame[f],
                    force=(f % 50 == 49)) for f in range(st.frame_count)]
    assert got == want
    assert len(db) == p.capacity and any(full for _, full in got)
    for i, pose in enumerate(ref.poses):
        assert np.array_equal(db.pose(i), pose) and np.array_equal(db.code(i), ref.codes[i])
    db.reset()
    assert len(db) == 0


def test_two_runs_are_identical(small_stream):
    st = small_stream
    rec = make(SMALL)
    p = with_(add_fraction=0.1)
    a_db, a = run_adds(st, p, rec)
    b_db, b = run_adds(st, p, rec)
    assert a == b and len(a_db) == len(b_db)
    for i in range(len(a_db)):
        assert np.array_equal(a_db.code(i), b_db.code(i))
    for f in (5, 77, 200):
        assert [x.tolist() for x in a_db.query(st.depth[f], st.color[f])] == \
               [x.tolist() for x in b_db.query(st.depth[f], st.color[f])]
        assert torch.equal(a_db.encode(st.depth[f], st.color[f]), b_db.encode(st.depth[f], st.color[f]))


# ---- relocalisation --------------------------------------------------------------------------------------------------

MAPPED = 150


@pytest.fixture(scope="module")
def mapped():
    """The cloud of the first 150 frames of the VGA desk stream integrated with their true poses, and a database of
    those frames offered at their true poses with the default params."""
    st = S.make_stream(VGA, MAPPED, device="cuda")
    pp, ip = params(VGA)
    rec = make()
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    db = R.KeyframeDatabase(rec)
    for f in range(first, last):
        db.add(st.depth[f], st.color[f], st.global_T_frame[f], depth_scaling=pp.depth_scaling)
    torch.cuda.synchronize()
    return st, rec, db


REVISITS = [20, 45, 70, 95]


@pytest.fixture(scope="module")
def revisits():
    return W.revisit_frames(VGA, REVISITS)


def cloud_params():
    tp = _lib.TrackParams.from_buffer_copy(RelocParams.defaults().track)
    tp.model_source = _lib.TRACK_CLOUD
    return tp


@pytest.mark.parametrize("rgbd", [False, True], ids=["depth", "rgbd"])
def test_accepted_pose_is_the_tracking_call_from_that_keyframe(mapped, revisits, rgbd):
    st, rec, db = mapped
    pp, _ = params(VGA)
    rp = TrackRGBDParams.defaults() if rgbd else None
    depth, color, truth = revisits[1]
    pose, res = rec.relocalise(db, depth, color, rgbd=rp, pp=pp)
    assert res.relocalised == 1 and res.attempts == res.rank + 1 and 0 <= res.keyframe < len(db)
    idx, dist = db.query(depth, color)
    assert idx[res.rank] == res.keyframe and dist[res.rank] == res.distance
    if rgbd:
        again, tr = rec.track_rgbd(depth, color, db.pose(res.keyframe), params=cloud_params(), rgbd=rp, pp=pp)
        tr = tr.depth
    else:
        again, tr = rec.track(depth, db.pose(res.keyframe), params=cloud_params(), pp=pp)
    assert np.array_equal(pose.view(np.uint32), again.view(np.uint32))
    assert bytes(tr) == bytes(res.track)
    # the handle's previous frame is the accepted call's: a previous-frame track after sm_relocalise equals one after
    # that same tracking call
    nxt_depth, nxt_color, nxt_truth = revisits[1][0], revisits[1][1], truth
    guess = TW.compose(nxt_truth, offset((0.3, 0, 0), (0.004, 0, 0))).astype(np.float32)
    rec.relocalise(db, depth, color, rgbd=rp, pp=pp)
    if rgbd:
        a, ra = rec.track_rgbd(nxt_depth, nxt_color, guess, rgbd=rp, pp=pp, source="previous")
        rec.track_rgbd(depth, color, db.pose(res.keyframe), params=cloud_params(), rgbd=rp, pp=pp)
        b, rb = rec.track_rgbd(nxt_depth, nxt_color, guess, rgbd=rp, pp=pp, source="previous")
    else:
        a, ra = rec.track(nxt_depth, guess, pp=pp, source="previous")
        rec.track(depth, db.pose(res.keyframe), params=cloud_params(), pp=pp)
        b, rb = rec.track(nxt_depth, guess, pp=pp, source="previous")
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and bytes(ra) == bytes(rb)


def test_relocalisation_only_reads_the_state(mapped, revisits):
    st, rec, db = mapped
    pp, _ = params(VGA)
    before, n0, m0 = rec.dump_state()
    before = before.copy()
    count = len(db)
    for depth, color, _ in revisits[:2]:
        rec.relocalise(db, depth, color, pp=pp)
        rec.relocalise(db, depth, color, rgbd=TrackRGBDParams.defaults(), pp=pp)
    after, n1, m1 = rec.dump_state()
    assert (n0, m0) == (n1, m1) and np.array_equal(before.view(np.uint32), after.view(np.uint32))
    assert len(db) == count


def test_launch_counts(product, mapped, revisits):
    st, rec, db = mapped
    pp, _ = params(VGA)
    launches = product.fn["kernel_launch_count"]
    depth, color, truth = revisits[2]
    empty = R.KeyframeDatabase(rec)
    torch.cuda.synchronize()
    n0 = launches()
    pose, res = rec.relocalise(empty, depth, color, pp=pp)
    query_launches = launches() - n0
    assert res.relocalised == 0 and res.attempts == 0 and np.isnan(pose).all() and res.keyframe == -1
    assert query_launches == 4   # median downscale, encode, distance, select: no tracking launch
    n0 = launches()
    rec.track(depth, truth, params=cloud_params(), pp=pp)
    per_track = launches() - n0
    # every attempt fails with an impossible RMS bound: the most attempts, each one tracking call
    strict = with_(accept_rms=0.0, candidates=5)
    n0 = launches()
    pose, res = rec.relocalise(db, depth, color, params=strict, pp=pp)
    assert res.relocalised == 0 and np.isnan(pose).all()
    assert 1 <= res.attempts <= 5
    assert launches() - n0 == query_launches + res.attempts * per_track
    n0 = launches()
    pose, res = rec.relocalise(db, depth, color, pp=pp)
    assert res.relocalised == 1 and launches() - n0 == query_launches + res.attempts * per_track
    n0 = launches()
    db.query(depth, color)
    db.add(depth, color, truth)
    assert launches() - n0 == 8
    empty.close()


def test_invalid_arguments_are_rejected_without_a_launch(product, mapped):
    st, rec, db = mapped
    pp, _ = params(VGA)
    launches = product.fn["kernel_launch_count"]
    fn = rec.lib.fn
    bad = _lib.SM_ERR_INVALID_ARGUMENT
    depth, color = st.depth[10], st.color[10]
    dp, cp = depth.data_ptr(), color.data_ptr()
    I = np.eye(4, dtype=np.float32)[:3].copy()
    out = np.zeros(12, np.float32)
    codes = torch.zeros(64, dtype=torch.int32, device="cuda")
    other = make(SMALL)
    tiny = R.CUDASurfelReconstruction(1000, 20, 15, 20.0, 20.0, 10.0, 7.5)
    torch.cuda.synchronize()
    n0 = launches()
    h = C.c_void_p()
    nan, inf = float("nan"), float("inf")
    for field, value in [("level", 0), ("level", 5), ("ferns", 12), ("ferns", 0), ("ferns", 2056), ("min_depth", nan),
                         ("min_depth", 5.0), ("max_depth", inf), ("capacity", 0), ("add_fraction", 1.5),
                         ("add_fraction", nan), ("candidates", 0), ("candidates", 9), ("max_query_fraction", -0.1),
                         ("accept_inlier_fraction", 2.0), ("accept_rms", nan), ("accept_rms", -1.0)]:
        assert fn["keyframe_db_create"](C.byref(h), rec._h, C.byref(with_(**{field: value}))) == bad, field
    tp = with_()
    tp.track.levels = 5
    assert fn["keyframe_db_create"](C.byref(h), rec._h, C.byref(tp)) == bad
    assert fn["keyframe_db_create"](C.byref(h), tiny._h, C.byref(with_(level=4))) == bad   # blocks 20 x 15 > 16
    assert fn["keyframe_db_create"](None, rec._h, C.byref(with_())) == bad
    row, crow = 2 * VGA.width, 3 * VGA.width
    enc = lambda d=dp, dpitch=row, c=cp, cpitch=crow, s=5000.0, o=codes.data_ptr(): fn["keyframe_db_encode"](
        db._h, None, d, dpitch, c, cpitch, s, o)
    assert enc(d=None) == bad and enc(c=None) == bad and enc(o=None) == bad
    assert enc(dpitch=row - 1) == bad and enc(cpitch=crow - 1) == bad and enc(s=0.0) == bad and enc(s=nan) == bad
    i32, f32 = C.c_int32(), C.c_int32()
    for k in range(12):
        g = I.copy().reshape(-1)
        g[k] = nan
        assert fn["keyframe_db_add"](db._h, None, dp, row, cp, crow, 5000.0, g.ctypes.data_as(C.c_void_p), 0,
                                     C.byref(i32), C.byref(f32)) == bad
    mirrored = I.copy()
    mirrored[0, 0] = -1.0
    assert fn["keyframe_db_add"](db._h, None, dp, row, cp, crow, 5000.0, mirrored.ctypes.data_as(C.c_void_p), 0,
                                 C.byref(i32), C.byref(f32)) == bad
    assert fn["keyframe_db_add"](db._h, None, dp, row, cp, crow, 5000.0, I.ctypes.data_as(C.c_void_p), 0, None,
                                 C.byref(f32)) == bad
    idx, dist = np.zeros(8, np.int32), np.zeros(8, np.uint32)
    assert fn["keyframe_db_query"](db._h, None, dp, row - 2, cp, crow, 5000.0, idx.ctypes.data_as(C.c_void_p),
                                   dist.ctypes.data_as(C.c_void_p), C.byref(i32)) == bad
    assert fn["keyframe_db_read"](db._h, len(db), out.ctypes.data_as(C.c_void_p), None) == bad
    res = RelocResult()
    rel = lambda r=rec._h, p=None, ppx=pp, d=dp, dpitch=row, c=cp, cpitch=crow, rp=None: fn["relocalise"](
        r, db._h, None, C.byref(p) if p is not None else None, C.byref(ppx), C.byref(rp) if rp is not None else None,
        d, dpitch, c, cpitch, out.ctypes.data_as(C.c_void_p), C.byref(res))
    assert rel(r=other._h) == bad                                  # a handle of another camera size
    assert rel(d=None) == bad and rel(c=None) == bad and rel(dpitch=row - 1) == bad and rel(cpitch=crow - 1) == bad
    assert rel(p=with_(ferns=256)) == bad and rel(p=with_(seed=1)) == bad and rel(p=with_(capacity=5)) == bad
    assert rel(p=with_(candidates=0)) == bad and rel(p=with_(accept_rms=nan)) == bad
    pp_bad = PreprocessParams.from_buffer_copy(pp)
    pp_bad.depth_scaling = 0.0
    assert rel(ppx=pp_bad) == bad
    rp_bad = TrackRGBDParams.defaults()
    rp_bad.photometric_weight = -1.0
    assert rel(rp=rp_bad) == bad
    torch.cuda.synchronize()
    assert launches() == n0
    assert rel() == _lib.SM_OK and rel(p=with_(candidates=1, accept_rms=0.02)) == _lib.SM_OK
    tiny.close()
    other.close()


def test_relocalisation_during_a_session(mapped, revisits):
    """Relocalisation is allowed while a stream session is open, like tracking."""
    st, rec0, db0 = mapped
    pp, ip = params(VGA)
    rec = make()
    db = R.KeyframeDatabase(rec)
    with rec.session(pp, ip, (VGA.width, VGA.height)) as s:
        for f in range(40):
            status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            if status.last_integrated_frame >= 0:
                db.add(st.depth[f], st.color[f], st.global_T_frame[f], stream=s.stream)
        depth, color, truth = W.revisit_frames(VGA, [25])[0]
        pose, res = rec.relocalise(db, depth, color, pp=pp, stream=s.stream)
        assert res.relocalised == 1
        dt, dr = TW.pose_error(pose, truth)
        assert dt <= MAX_T and dr <= MAX_R


# ---- kidnapped camera ------------------------------------------------------------------------------------------------

def test_kidnapped_camera(mapped, revisits):
    """Frames that come back to mapped places, a few cm and degrees off every pushed pose, with noise of their own:
    the tracker from the pose before the jump reports them lost, sm_relocalise recovers them within the pose-free
    bounds, and frames of the never-mapped far side of the orbit are not accepted at a wrong pose."""
    st, rec, db = mapped
    pp, _ = params(VGA)
    pre_jump = st.global_T_frame[MAPPED - 1]
    report = []
    for (depth, color, truth), f in zip(revisits, REVISITS):
        nearest = min(TW.pose_error(truth, st.global_T_frame[g]) for g in range(MAPPED))
        assert nearest[0] > 0.005 or nearest[1] > 0.3   # not a repeat of a mapped frame
        _, tr = rec.track(depth, pre_jump, pp=pp)
        assert tr.tracked == 0, f
        pose, res = rec.relocalise(db, depth, color, pp=pp)
        assert res.relocalised == 1, (f, res.attempts)
        dt, dr = TW.pose_error(pose, truth)
        report.append((f, res.attempts, res.keyframe, dt * 1e3, dr))
        assert dt <= MAX_T and dr <= MAX_R, (f, dt, dr)
    far = S.trajectory(601)
    accepted = 0
    for k in (420, 480, 540, 600):
        depth, color = W.render_frame(VGA, far[k], 900 + k)
        pose, res = rec.relocalise(db, depth, color, pp=pp)
        if res.relocalised:
            accepted += 1
            dt, dr = TW.pose_error(pose, far[k])
            assert dt <= MAX_T and dr <= MAX_R, ("accepted a wrong pose", k, dt, dr)
    print(f"kidnapped: {report}; unmapped accepted {accepted}/4")


def jump_session(reloc):
    """Frames 0-149 of the desk stream, then a jump back to orbit frames 60-79 (moved 1.5 cm / 1.1 degrees, fresh
    noise), through a TrackedSession."""
    st = S.make_stream(VGA, MAPPED, device="cuda")
    tail = W.jump_frames(VGA, 60, 20)
    pp, ip = params(VGA)
    rec = make()
    truth = list(st.global_T_frame) + [p for _, _, p in tail]
    with R.TrackedSession(rec, pp, ip, st.global_T_frame[0], reloc=reloc) as s:
        for f in range(MAPPED):
            s.push(st.depth[f], st.color[f])
        for depth, color, _ in tail:
            s.push(depth, color)
    return s, truth


def test_pose_free_session_relocalises_after_a_jump():
    s, truth = jump_session(RelocParams.defaults())
    states = s.states
    assert states[:MAPPED] == ["tracked"] * MAPPED
    after = states[MAPPED:]
    k = after.index("relocalised")
    assert all(x == "lost" for x in after[:k]) and k <= 2
    assert after[k + 1:] == ["tracked"] * (len(after) - k - 1)
    pushed = [f for f, x in enumerate(states) if x != "lost"]
    errors = np.array([TW.pose_error(s.trajectory[f], truth[f]) for f in pushed])
    print(f"jump with relocalisation: states after the jump {after}, max {errors[:, 0].max() * 1e3:.2f} mm / "
          f"{errors[:, 1].max():.3f} deg, {len(s.database)} keyframes")
    assert errors[:, 0].max() <= MAX_T and errors[:, 1].max() <= MAX_R
    held = [f for f, x in enumerate(states) if x == "lost"]
    assert all(np.isnan(s.trajectory[f]).all() for f in held)
    assert len(s.trajectory) == len(truth) and len(s.database) > 0


def test_pose_free_session_without_relocalisation_pushes_wrong_poses():
    """The failure relocalisation fixes: the same stream without it pushes the frames after the jump at poses far
    from the truth."""
    s, truth = jump_session(None)
    errors = np.array([TW.pose_error(s.trajectory[f], truth[f]) for f in range(MAPPED, len(truth))])
    assert s.states[MAPPED] == "lost" and not np.isnan(s.trajectory[MAPPED]).any()   # pushed at its guess
    assert errors[:, 0].max() > 0.1


def test_pose_free_stream_without_loss_never_relocalises():
    st = S.make_stream(VGA, 120, device="cuda")
    pp, ip = params(VGA)
    rec = make()
    with R.TrackedSession(rec, pp, ip, st.global_T_frame[0], reloc=RelocParams.defaults()) as s:
        for f in range(st.frame_count):
            s.push(st.depth[f], st.color[f])
    assert s.states == ["tracked"] * st.frame_count and all(r is None for r in s.reloc_results)
    assert len(s.database) > 0
    errors = np.array([TW.pose_error(s.trajectory[f], st.global_T_frame[f]) for f in range(st.frame_count)])
    print(f"no loss: {len(s.database)} keyframes, max {errors[:, 0].max() * 1e3:.2f} mm / {errors[:, 1].max():.3f} deg")
    assert errors[:, 0].max() <= MAX_T and errors[:, 1].max() <= MAX_R
