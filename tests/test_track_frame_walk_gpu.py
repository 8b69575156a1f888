"""sm_track_frame / sm_track_frame_rgbd held bit for bit to the frame walk of tests/track_walk.py: the device's own
system of every Gauss-Newton step (sm_track_linearize*, itself checked against the restated linearisation) through
the restated solve, SE(3) update, loss and convergence rules, level schedule and pose bookkeeping. global_T_out,
tracked, iterations, inliers, valid_pixels (and photometric_inliers, rms_intensity) must match exactly, rms_residual
within 1 ulp (its sum r^2 is the restatement's, in another order). A frame with a step whose fp32 rounding the
device's sin / cos could tip (the clear rule of track_walk.solve_step) is excused and counted."""
import math
import time

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, TrackParams, TrackRGBDParams
from tests import track_rgbd_walk as RW
from tests import track_walk as TW
from tests.util import offset

pytestmark = pytest.mark.gpu

VGA = S.Camera.tum(640, 480)
ODD = S.Camera.tum(321, 243)   # Camera.scaled sizes round up at level 1 (161 x 122) and down at level 3 (40 x 30)
QVGA = S.Camera.tum(320, 240)
CAP = 2_000_000
TILT_5 = tuple(5.0 * np.array([3.0, -2.6, 2.9]) / np.linalg.norm([3.0, -2.6, 2.9]))
START = time.perf_counter()
COMPARED, EXCUSED = [], []   # the case names of the frames compared and of the frames excused by the clear rule


def make(cam):
    return R.CUDASurfelReconstruction(CAP, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


def pre(cam):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    return pp


def schedule(levels=3, iterations=(4, 5, 10, 0), **fields):
    tp = TrackParams.defaults()
    tp.levels = levels
    tp.iterations = (type(tp.iterations))(*iterations)
    for k, v in fields.items():
        setattr(tp, k, v)
    return tp


def integrate(cam, frames):
    st = S.make_stream(cam, frames, device="cuda")
    rec = make(cam)
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pre(cam),
                   IntegrateParams.defaults(), first, last)
    torch.cuda.synchronize()
    return st, rec


@pytest.fixture(scope="module")
def vga():
    """The cloud after 40 integrated frames of the VGA synthetic stream."""
    return integrate(VGA, 48)


@pytest.fixture(scope="module")
def odd():
    """The cloud after 16 integrated frames of the synthetic stream at 321 x 243."""
    return integrate(ODD, 24)


def device_call(rec, depth, guess, tp, pp, source, color, rp):
    if color is None:
        out, res = rec.track(depth, guess, params=tp, pp=pp, source=source)
        return out, res, None
    out, res = rec.track_rgbd(depth, color, guess, params=tp, rgbd=rp, pp=pp, source=source)
    return out, res.depth, res


def differences(pred, out, res, rgbd_res):
    bits = lambda a: np.asarray(a, np.float32).reshape(-1).view(np.int32)
    diff = []
    if not np.array_equal(bits(out), bits(pred["pose"])):
        diff.append(("pose", out.reshape(-1).tolist(), pred["pose"].reshape(-1).tolist()))
    for name in ("tracked", "iterations", "inliers", "valid_pixels"):
        if getattr(res, name) != pred[name]:
            diff.append((name, getattr(res, name), pred[name]))
    if abs(int(bits(res.rms_residual)[0]) - int(bits(pred["rms_residual"])[0])) > 1:
        diff.append(("rms_residual", res.rms_residual, float(pred["rms_residual"])))
    if rgbd_res is not None:
        if rgbd_res.photometric_inliers != pred["photometric_inliers"]:
            diff.append(("photometric_inliers", rgbd_res.photometric_inliers, pred["photometric_inliers"]))
        if bits(rgbd_res.rms_intensity)[0] != bits(pred["rms_intensity"])[0]:
            diff.append(("rms_intensity", rgbd_res.rms_intensity, float(pred["rms_intensity"])))
    return diff


def first_differing_step(rec, depth, guess, tp, pp, color=None, rp=None):
    """For a SM_TRACK_CLOUD call that differs from the walk: sm_track_frame re-run on the schedule truncated after each
    scheduled step in turn, against the walk's prediction for the same prefix. Returns the first (level, steps at
    that level, differences), or None if every prefix agrees."""
    for level in range(tp.levels - 1, -1, -1):
        for k in range(1, tp.iterations[level] + 1):
            iters = [tp.iterations[l] if l > level else (k if l == level else 0) for l in range(4)]
            t = TrackParams.from_buffer_copy(tp)
            t.iterations = (type(t.iterations))(*iters)
            pred = TW.track_frame(rec, depth, guess, t, pp, "cloud", None, color, rp)
            out, res, rgbd_res = device_call(rec, depth, guess, t, pp, "cloud", color, rp)
            diff = differences(pred, out, res, rgbd_res)
            if diff:
                return level, k, diff
    return None


def check(case, rec, depth, guess, tp, pp, source="cloud", previous=None, color=None, rp=None):
    """One tracking call on the device and in the walk; returns the walk's prediction."""
    guess = np.asarray(guess, np.float32).reshape(3, 4)
    pred = TW.track_frame(rec, depth, guess, tp, pp, source, previous, color, rp)
    out, res, rgbd_res = device_call(rec, depth, guess, tp, pp, source, color, rp)
    if not pred["clear"]:
        EXCUSED.append(case)
        return pred
    COMPARED.append(case)
    diff = differences(pred, out, res, rgbd_res)
    if diff and source == "cloud":
        diff.append(("first differing step", first_differing_step(rec, depth, guess, tp, pp, color, rp)))
    assert not diff, (case, diff)
    return pred


GUESSES = {"exact": ((0, 0, 0), (0, 0, 0)), "2cm_2deg": ((1.2, -1.1, 1.15), (0.012, -0.011, 0.0115)),
           "5cm": ((0, 0, 0), (0.03, -0.03, 0.026)), "tilt_5deg": (TILT_5, (0, 0, 0))}
SCHEDULES = {"default": (4, 5, 10, 0), "sparse": (0, 3, 0, 2), "ones": (1, 1, 1, 1)}


def schedule_case(st, rec, cam, levels, sched, guess_name, frame=31):
    tp = schedule(levels, SCHEDULES[sched])
    guess = TW.compose(st.global_T_frame[frame], offset(*GUESSES[guess_name])).astype(np.float32)
    pred = check(f"{cam.width}x{cam.height} levels {levels} {sched} {guess_name}", rec, st.depth[frame].cuda(), guess,
                 tp, pre(cam))
    if tp.iterations[0] == 0:   # no level-0 step: the level-0 statistics stay 0
        assert pred["inliers"] == pred["valid_pixels"] == 0
    if guess_name == "tilt_5deg" and tp.iterations[tp.levels - 1] > 0:
        assert pred["tracked"] == 0
    return pred


@pytest.mark.parametrize("sched", sorted(SCHEDULES))
@pytest.mark.parametrize("levels", [1, 2, 3, 4])
def test_schedules_vga(vga, levels, sched):
    st, rec = vga
    schedule_case(st, rec, VGA, levels, sched, "2cm_2deg")


@pytest.mark.parametrize("guess_name", ["exact", "5cm", "tilt_5deg"])
@pytest.mark.parametrize("sched", sorted(SCHEDULES))
@pytest.mark.parametrize("levels", [3, 4])
def test_guesses_vga(vga, levels, sched, guess_name):
    st, rec = vga
    schedule_case(st, rec, VGA, levels, sched, guess_name)


@pytest.mark.parametrize("sched", sorted(SCHEDULES))
@pytest.mark.parametrize("levels", [1, 2, 3, 4])
def test_schedules_odd_size(odd, levels, sched):
    st, rec = odd
    schedule_case(st, rec, ODD, levels, sched, "2cm_2deg", frame=13)


def norms(step):
    xi = step["xi"]
    return math.sqrt(xi[0] ** 2 + xi[1] ** 2 + xi[2] ** 2), math.sqrt(xi[3] ** 2 + xi[4] ** 2 + xi[5] ** 2)


def test_convergence_ends_the_chosen_level(vga):
    """Thresholds taken from the walk's own step norms on the coarsest level (twice the chosen step's, and at most
    half of one of the previous step's): that level ends after the chosen step, on the device as in the walk, and
    more iterations on it change nothing."""
    st, rec = vga
    pp = pre(VGA)
    depth = st.depth[31].cuda()
    guess = TW.compose(st.global_T_frame[31], offset(*GUESSES["5cm"])).astype(np.float32)
    free = TW.track_frame(rec, depth, guess, schedule(convergence_rotation=0.0, convergence_translation=0.0), pp)
    coarse = [s for s in free["trace"] if s["level"] == 2 and not s["skipped"]]
    chosen = None
    for k in (2, 3, 1, 4, 5):
        w, v = norms(coarse[k])
        cr, ct = float(np.float32(2 * w)), float(np.float32(2 * v))
        if all(norms(coarse[j])[0] > 2 * cr or norms(coarse[j])[1] > 2 * ct for j in range(k)):
            chosen = k, cr, ct
            break
    assert chosen, [norms(s) for s in coarse]
    k, cr, ct = chosen
    tp = schedule(convergence_rotation=cr, convergence_translation=ct)
    pred = check("convergence", rec, depth, guess, tp, pp)
    at = [s for s in pred["trace"] if s["level"] == 2]
    assert [s["skipped"] for s in at] == [False] * (k + 1) + [True] * (10 - k - 1)
    assert at[k]["converged"] and not any(s["converged"] for s in at[:k])
    longer = schedule(3, (4, 5, 30, 0),convergence_rotation=cr, convergence_translation=ct)
    check("convergence, 30 coarse iterations", rec, depth, guess, longer, pp)
    a, ra = rec.track(depth, guess, params=tp, pp=pp)
    b, rb = rec.track(depth, guess, params=longer, pp=pp)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and bytes(ra) == bytes(rb)


def test_loss_at_the_inlier_fraction_boundary(vga):
    """min_inlier_fraction at the two fp32 values around inliers / valid of the first coarse linearisation: the
    double comparison inliers < fraction * valid flips between them. The guess is off SO(3), so the lost frame
    visibly returns it unprojected."""
    st, rec = vga
    pp = pre(VGA)
    depth = st.depth[31].cuda()
    guess = TW.compose(st.global_T_frame[31], offset((0.5, 0, 0), (0.005, 0, 0))).astype(np.float32)
    guess[:, :3] *= np.float32(1.002)
    guess[0, 1] += np.float32(0.001)
    first = TW.track_frame(rec, depth, guess, schedule(), pp)["trace"][0]["linearization"]
    inliers, valid = first["inliers"], first["valid"]
    lost_at = np.float32(inliers / valid)
    while not inliers < float(lost_at) * valid:
        lost_at = np.nextafter(lost_at, np.float32(1))
    kept_at = np.nextafter(lost_at, np.float32(0))
    while inliers < float(kept_at) * valid:
        kept_at = np.nextafter(kept_at, np.float32(0))
    assert np.nextafter(kept_at, np.float32(1)) == lost_at
    pred = check("fraction just above", rec, depth, guess, schedule(min_inlier_fraction=float(lost_at)), pp)
    assert pred["tracked"] == 0 and pred["trace"][0]["reason"] == "inliers" and pred["iterations"] == 0
    assert np.array_equal(pred["pose"], guess)
    pred = check("fraction just below", rec, depth, guess, schedule(min_inlier_fraction=float(kept_at)), pp)
    assert not pred["trace"][0]["lost"]


def test_zero_pivot_when_the_model_view_is_empty(vga):
    """A guess 1 km ahead of the camera sees no surfel: with min_inlier_fraction 0 the loss rule passes 0 of the
    valid pixels, and the zero system is lost by its first Cholesky pivot at the coarsest level."""
    st, rec = vga
    pp = pre(VGA)
    guess = TW.compose(st.global_T_frame[31], offset((0, 0, 0), (0, 0, 1000.0))).astype(np.float32)
    pred = check("zero pivot", rec, st.depth[31].cuda(), guess, schedule(min_inlier_fraction=0.0), pp)
    assert pred["trace"][0]["reason"] == "pivot" and pred["trace"][0]["level"] == 2
    assert pred["tracked"] == 0 and pred["iterations"] == 0 and pred["inliers"] == pred["valid_pixels"] == 0
    assert np.array_equal(pred["pose"], guess)


def constant_velocity(poses):
    if len(poses) < 2:
        return poses[-1]
    return TW.compose(TW.compose(poses[-1], TW.invert(poses[-2])), poses[-1]).astype(np.float32)


def chain(st, rec, rgbd, lost_call=3):
    """Six frames: the first against the cloud from its true pose, the others against the previous frame from the
    constant-velocity guess of the returned poses; call `lost_call`'s guess is turned by 5 degrees and lost, so the
    next call's model pose is that guess."""
    pp = pre(VGA)
    rp = TrackRGBDParams.defaults() if rgbd else None
    returned, previous, tracked = [], None, []
    for k, f in enumerate(range(30, 36)):
        color = st.color[f].cuda() if rgbd else None
        guess = st.global_T_frame[f] if k == 0 else constant_velocity(returned)
        if k == lost_call:
            guess = TW.compose(guess, offset(TILT_5, (0, 0, 0))).astype(np.float32)
        source = "cloud" if k == 0 else "previous"
        pred = check(f"{'rgbd' if rgbd else 'depth'} chain call {k}", rec, st.depth[f].cuda(), guess, schedule(), pp,
                     source, previous, color, rp)
        returned.append(pred["pose"])
        previous = pred["kept"]
        tracked.append(pred["tracked"])
    # the calls after the lost one start from its guess as the model pose, with the turn in their constant-velocity
    # guesses: they may be lost as well, which the walk has predicted call by call
    assert tracked[:lost_call] == [1] * lost_call and tracked[lost_call] == 0, tracked
    return previous


def test_previous_frame_chain_depth(vga):
    st, rec = vga
    chain(st, rec, rgbd=False)


def test_previous_frame_chain_rgbd(vga):
    st, rec = vga
    previous = chain(st, rec, rgbd=True)
    pp, rp = pre(VGA), TrackRGBDParams.defaults()
    # a depth-only call in between: the next RGB-D call may not track against the previous frame
    pred = check("depth call after the rgbd chain", rec, st.depth[36].cuda(), previous["pose"], schedule(), pp,
                 "previous", previous)
    with pytest.raises(_lib.SurfelError):
        rec.track_rgbd(st.depth[37].cuda(), st.color[37].cuda(), pred["pose"], rgbd=rp, pp=pp, source="previous")
    with pytest.raises(ValueError):
        TW.track_frame(rec, st.depth[37].cuda(), pred["pose"], schedule(), pp, "previous", pred["kept"],
                       st.color[37].cuda(), rp)


@pytest.mark.parametrize("levels,sched", [(3, "default"), (4, "sparse"), (4, "ones")])
def test_rgbd_against_the_cloud(vga, levels, sched):
    st, rec = vga
    guess = TW.compose(st.global_T_frame[32], offset(*GUESSES["2cm_2deg"])).astype(np.float32)
    pred = check(f"rgbd cloud levels {levels} {sched}", rec, st.depth[32].cuda(), guess,
                 schedule(levels, SCHEDULES[sched]), pre(VGA), color=st.color[32].cuda(), rp=TrackRGBDParams.defaults())
    if SCHEDULES[sched][0]:
        assert pred["photometric_inliers"] > 0


def test_rgbd_on_the_textured_wall():
    """One textured wall: depth alone leaves the slide along the wall free, colour fixes it."""
    depth, color, poses = RW.wall_stream((QVGA.width, QVGA.height, QVGA.fx, QVGA.fy, QVGA.cx, QVGA.cy), 40)
    depth = torch.from_numpy(depth.astype(np.int32)).to(torch.uint16).cuda()
    color = torch.from_numpy(color).cuda()
    g = poses.astype(np.float32)
    rec = make(QVGA)
    pp = pre(QVGA)
    rec.stream_run(None, depth, color, g, S.invert_poses(poses).astype(np.float32), S.others_TR_reference(poses, 5000.0, 8),
                   pp, IntegrateParams.defaults(), 4, 36)
    torch.cuda.synchronize()
    slide = np.concatenate([Rotation.from_rotvec(np.radians(1.0) * np.array([0, 0, 1.0])).as_matrix(),
                            np.array([[0.01], [-0.006], [0.0]])], axis=1)
    guess = TW.compose(slide, g[34]).astype(np.float32)
    pred = check("textured wall", rec, depth[34], guess, schedule(), pp, color=color[34], rp=TrackRGBDParams.defaults())
    assert pred["tracked"] == 1 and pred["photometric_inliers"] > 0


def test_excused_frames_are_rare():
    """Runs last: the frames the clear rule excused, of all the module compared (estimated far below one)."""
    print(f"\nframe walk: {len(COMPARED)} frames compared bit for bit, {len(EXCUSED)} excused {EXCUSED}, "
          f"{time.perf_counter() - START:.1f} s")
    assert len(EXCUSED) <= 1
