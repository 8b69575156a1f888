"""sm_track_frame / sm_track_linearize on the GPU: the linearisation against the numpy restatement
(tests/track_walk.py), pose recovery on exact data, pose-free synthetic streams (TrackedSession), determinism,
read-only behaviour, lost frames and argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import PreprocessParams, TrackParams, TrackResult
from tests import track_walk as TW
from tests.util import offset, params

pytestmark = pytest.mark.gpu

VGA = S.Camera.tum(640, 480)
SMALL = S.Camera.tum(160, 120)
CAP = 2_000_000
SCALE = 5000.0


def cam_tuple(cam):
    return (cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


def make(cam=VGA):
    return R.CUDASurfelReconstruction(CAP, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


pose_error = TW.pose_error


def assert_parity(rec, level, live, model_depth, model_normal, T, cam):
    lc = TW.scaled(cam_tuple(cam), level)
    live_t = torch.from_numpy(live.astype(np.int32)).to(torch.uint16).cuda()
    system, inliers = rec.track_linearize(level, live_t, torch.from_numpy(model_depth).cuda(),
                                          torch.from_numpy(np.ascontiguousarray(model_normal)).cuda(), T)
    ref = TW.linearize(live, SCALE, lc[2:], model_depth, model_normal, cam_tuple(cam)[2:], np.asarray(T, np.float32))
    assert inliers == ref["inliers"]
    assert inliers > 0
    bound = 1e-9 * ref["magnitude"] + 1e-300
    bad = np.abs(system - ref["system"]) > bound
    assert not bad.any(), (np.flatnonzero(bad), system[bad], ref["system"][bad])


OFFSETS = {"identity": ((0, 0, 0), (0, 0, 0)), "small": ((0.3, -0.2, 0.4), (0.005, -0.004, 0.006)),
           "large": ((1.5, 1.0, -2.0), (0.02, 0.03, -0.025))}


@pytest.mark.parametrize("scene", sorted(TW.SCENES))
@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("off", sorted(OFFSETS))
def test_linearize_matches_restatement_on_planes(scene, level, off):
    cam = cam_tuple(SMALL)
    z, n = TW.render_planes(TW.SCENES[scene], cam, np.eye(4)[:3])
    model_depth = np.where(np.isfinite(z), z, 0).astype(np.float32)
    model_normal = n.astype(np.float32)
    model_depth[10:14, 20:30] = np.nan
    model_depth[40:44, 50:58] = 0
    model_normal[60:62, 60:70] = np.nan
    truth = offset((0.5, -0.8, 0.3), (0.01, 0.005, -0.01))
    zl, _ = TW.render_planes(TW.SCENES[scene], TW.scaled(cam, level), truth)
    live = TW.quantize(zl)
    live[3:6, 3:12] = 0
    rec = make(SMALL)
    assert_parity(rec, level, live, model_depth, model_normal, offset(*OFFSETS[off]).astype(np.float32), SMALL)


@pytest.fixture(scope="module")
def integrated():
    """The cloud after 40 integrated frames of the VGA synthetic stream."""
    st = S.make_stream(VGA, 48, device="cuda")
    pp, ip = params(VGA)
    rec = make()
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    torch.cuda.synchronize()
    return st, rec


def model_view(rec, global_T_camera):
    out = rec.render(R.invert_rigid(global_T_camera), VGA.width, VGA.height, VGA.fx, VGA.fy, VGA.cx, VGA.cy,
                     near=0.1, far=100.0, outputs=("depth", "normal"))
    torch.cuda.synchronize()
    return out["depth"].cpu().numpy(), out["normal"].cpu().numpy()


@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("off", sorted(OFFSETS))
def test_linearize_matches_restatement_on_a_rendered_cloud(integrated, level, off):
    st, rec = integrated
    model_depth, model_normal = model_view(rec, st.global_T_frame[30])
    # the live frame: the raw depth of frame 31, median-downscaled to the level as the tracker does
    raw = st.depth[31].cuda()
    lc = TW.scaled(cam_tuple(VGA), level)
    live = R.DownscaleUsingMedianWhileExcluding(None, 0, lc[0], lc[1], raw).cpu().numpy() if level else raw.cpu().numpy()
    rel = TW.compose(R.invert_rigid(st.global_T_frame[30]), st.global_T_frame[31])
    T = TW.compose(offset(*OFFSETS[off]), rel).astype(np.float32)
    assert_parity(rec, level, live, model_depth, model_normal, T, VGA)


def quantized_render(rec, global_T_camera):
    depth, _ = model_view(rec, global_T_camera)
    return torch.from_numpy(TW.quantize(depth.astype(np.float64), SCALE).astype(np.int32)).to(torch.uint16).cuda()


TILT_5 = tuple(5.0 * np.array([3.0, -2.6, 2.9]) / np.linalg.norm([3.0, -2.6, 2.9]))


@pytest.mark.parametrize("perturbation", [((1.2, -1.1, 1.15), (0.012, -0.011, 0.0115)), ((0, 0, 0), (0.03, -0.03, 0.026)),
                                          ((0, 0, 5.0), (0, 0, 0))], ids=["2cm_2deg", "5cm", "5deg_roll"])
def test_recovers_the_pose_of_exact_data(integrated, perturbation):
    st, rec = integrated
    pose = st.global_T_frame[30]
    live = quantized_render(rec, pose)
    guess = TW.compose(pose, offset(*perturbation)).astype(np.float32)
    t0, r0 = pose_error(guess, pose)
    assert t0 > 0.01 or r0 > 1.5
    pp, _ = params(VGA)
    out, res = rec.track(live, guess, pp=pp)
    dt, dr = pose_error(out, pose)
    print(f"exact data, start {t0 * 1000:.1f} mm / {r0:.2f} deg: {dt * 1000:.3f} mm, {dr:.4f} deg, "
          f"{res.iterations} steps, inliers {res.inliers}/{res.valid_pixels}, rms {res.rms_residual * 1000:.3f} mm")
    assert res.tracked == 1
    assert dt <= 1e-3 and dr <= 0.05


def test_a_five_degree_tilt_is_reported_lost(integrated):
    """A 5-degree rotation about an axis across the view leaves ~3 % of the valid live pixels within the 5 cm
    point-to-point gate (tests/test_track_host.py::test_five_degree_guesses_inlier_fraction measures it), below
    min_inlier_fraction: the tracker reports the frame lost and returns the guess instead of a wrong pose."""
    st, rec = integrated
    pose = st.global_T_frame[30]
    guess = TW.compose(pose, offset(TILT_5, (0, 0, 0))).astype(np.float32)
    assert abs(pose_error(guess, pose)[1] - 5.0) < 1e-3
    pp, _ = params(VGA)
    out, res = rec.track(quantized_render(rec, pose), guess, pp=pp)
    assert res.tracked == 0 and np.array_equal(out, guess)


def test_a_guess_off_so3_is_projected(integrated):
    """The rotation of the guess is replaced by its nearest rotation, and the returned pose is a rotation to fp32
    rounding: a chain of calls cannot accumulate scale or shear."""
    st, rec = integrated
    pose = st.global_T_frame[30]
    guess = TW.compose(pose, offset((0.5, 0, 0), (0.005, 0, 0))).astype(np.float32)
    guess[:, :3] *= np.float32(1.002)
    guess[0, 1] += np.float32(0.001)
    pp, _ = params(VGA)
    out, res = rec.track(quantized_render(rec, pose), guess, pp=pp)
    rot = out[:, :3].astype(np.float64)
    assert res.tracked == 1
    assert np.abs(rot @ rot.T - np.eye(3)).max() < 1e-6
    dt, dr = pose_error(out, pose)
    assert dt <= 1e-3 and dr <= 0.05


def test_two_calls_are_bit_identical(integrated):
    st, rec = integrated
    pp, _ = params(VGA)
    live = st.depth[32].cuda()
    guess = TW.compose(st.global_T_frame[32], offset((0.5, 0.5, 0), (0.01, 0, 0))).astype(np.float32)
    a, ra = rec.track(live, guess, pp=pp)
    b, rb = rec.track(live, guess, pp=pp)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert bytes(ra) == bytes(rb)
    assert ra.tracked == 1


def test_tracking_only_reads_the_state(integrated):
    st, rec = integrated
    pp, _ = params(VGA)
    before, n0, m0 = rec.dump_state()
    before = before.copy()
    rec.track(st.depth[33].cuda(), st.global_T_frame[33], pp=pp)
    rec.track(st.depth[34].cuda(), st.global_T_frame[34], pp=pp, source="previous")
    after, n1, m1 = rec.dump_state()
    assert (n0, m0) == (n1, m1)
    assert np.array_equal(before.view(np.uint32), after.view(np.uint32))


def test_lost_frames_return_the_guess(integrated):
    st, rec = integrated
    pp, _ = params(VGA)
    empty = make()
    guess = st.global_T_frame[20]
    out, res = empty.track(st.depth[20].cuda(), guess, pp=pp)
    assert res.tracked == 0 and np.array_equal(out, np.asarray(guess, np.float32))
    far = TW.compose(st.global_T_frame[20], offset((0, 0, 0), (0.0, 0.0, 1.0))).astype(np.float32)
    out, res = rec.track(st.depth[20].cuda(), far, pp=pp)
    assert res.tracked == 0 and np.array_equal(out, far)


def test_invalid_arguments_are_rejected_without_a_launch(product):
    rec = make(SMALL)
    pp, _ = params(SMALL)
    depth = torch.zeros((SMALL.height, SMALL.width), dtype=torch.uint16, device="cuda")
    md = torch.zeros((SMALL.height, SMALL.width), dtype=torch.float32, device="cuda")
    mn = torch.zeros((SMALL.height, SMALL.width, 3), dtype=torch.float32, device="cuda")
    I = np.eye(4, dtype=np.float32)[:3].copy()
    out = np.zeros(12, np.float32)
    sysv = np.zeros(27, np.float64)
    inl = C.c_uint32()
    fn = rec.lib.fn

    def frame(tp=None, ptr=depth.data_ptr(), pitch=2 * SMALL.width, guess=I, res=True, ppx=pp):
        tp = tp or TrackParams.defaults()
        r = TrackResult()
        return fn["track_frame"](rec._h, None, C.byref(tp), C.byref(ppx), ptr, pitch, guess.ctypes.data_as(C.c_void_p),
                                 out.ctypes.data_as(C.c_void_p), C.byref(r) if res else None)

    def lin(level=0, tp=None, scale=SCALE, live_pitch=2 * SMALL.width, depth_pitch=4 * SMALL.width,
            normal_pitch=12 * SMALL.width, T=I, live=depth.data_ptr()):
        tp = tp or TrackParams.defaults()
        return fn["track_linearize"](rec._h, None, C.byref(tp), level, scale, live, live_pitch, md.data_ptr(),
                                     depth_pitch, mn.data_ptr(), normal_pitch, T.ctypes.data_as(C.c_void_p),
                                     sysv.ctypes.data_as(C.c_void_p), C.byref(inl))

    def with_(**kw):
        tp = TrackParams.defaults()
        for k, v in kw.items():
            setattr(tp, k, v)
        return tp

    tiny = R.CUDASurfelReconstruction(1000, 4, 3, 3.0, 3.0, 2.0, 1.5)
    torch.cuda.synchronize()
    launches = product.fn["kernel_launch_count"]()
    bad = _lib.SM_ERR_INVALID_ARGUMENT
    nan, inf = float("nan"), float("inf")
    # the first call on a handle may not use the previous frame
    assert frame(with_(model_source=_lib.TRACK_PREVIOUS_FRAME)) == bad
    assert frame(ptr=None) == bad and frame(res=False) == bad and frame(pitch=2 * SMALL.width - 1) == bad
    for levels in (0, 5, -1):
        assert frame(with_(levels=levels)) == bad, levels
    assert frame(with_(iterations=(C.c_int32 * 4)(4, -1, 10, 0))) == bad
    for field, value in [("max_point_distance", nan), ("max_point_distance", 0.0), ("max_point_distance", inf),
                         ("max_normal_angle_deg", nan), ("min_inlier_fraction", nan), ("convergence_rotation", inf),
                         ("convergence_translation", nan), ("convergence_rotation", -1.0), ("model_source", 7)]:
        assert frame(with_(**{field: value})) == bad, field
    for k in range(12):
        g = I.copy().reshape(-1)
        g[k] = nan if k % 2 else inf
        assert frame(guess=g) == bad, k
    mirrored = I.copy()
    mirrored[0, 0] = -1.0
    assert frame(guess=mirrored) == bad
    pp_bad = PreprocessParams.from_buffer_copy(pp)
    pp_bad.depth_scaling = 0.0
    assert frame(ppx=pp_bad) == bad
    # a level too small for the image: 160 x 120 has 20 x 15 at level 3, a 4 x 3 handle has nothing past level 0
    tp2 = with_(levels=2)
    r = TrackResult()
    assert fn["track_frame"](tiny._h, None, C.byref(tp2), C.byref(pp), depth.data_ptr(), 8, I.ctypes.data_as(C.c_void_p),
                             out.ctypes.data_as(C.c_void_p), C.byref(r)) == bad
    for level in (-1, 4):
        assert lin(level=level) == bad, level
    assert lin(scale=0.0) == bad and lin(scale=nan) == bad and lin(live=None) == bad
    assert lin(live_pitch=2 * SMALL.width - 1) == bad and lin(depth_pitch=4 * SMALL.width - 1) == bad
    assert lin(normal_pitch=12 * SMALL.width - 1) == bad
    assert lin(level=1, live_pitch=SMALL.width - 1) == bad
    Tn = I.copy()
    Tn[1, 3] = nan
    assert lin(T=Tn) == bad and lin(tp=with_(max_point_distance=nan)) == bad
    # the Python wrapper checks the image sizes and types the C ABI cannot see
    for args in ((1, depth, md, mn), (0, depth.to(torch.int16), md, mn), (0, depth, md[:, :-1], mn),
                 (0, depth, md, mn[..., :2]), (0, depth, md.double(), mn), (4, depth, md, mn)):
        with pytest.raises(ValueError):
            rec.track_linearize(args[0], *args[1:], I)
    torch.cuda.synchronize()
    assert product.fn["kernel_launch_count"]() == launches
    # and valid calls still work on the same handle
    assert lin(level=1, live_pitch=SMALL.width) == _lib.SM_OK
    assert frame() == _lib.SM_OK
    assert frame(with_(model_source=_lib.TRACK_PREVIOUS_FRAME)) == _lib.SM_OK


def test_tracking_between_session_pushes():
    st = S.make_stream(VGA, 30, device="cuda")
    pp, ip = params(VGA)
    rec = make()
    tracked = []
    with rec.session(pp, ip, (VGA.width, VGA.height)) as s:
        for f in range(st.frame_count):
            status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            if f in (15, 25):
                assert status.last_integrated_frame >= 0
                guess = TW.compose(st.global_T_frame[f], offset((0.5, 0, 0), (0.01, 0, 0))).astype(np.float32)
                out, res = rec.track(st.depth[f].cuda(), guess, pp=pp, stream=s.stream)
                dt, dr = pose_error(out, st.global_T_frame[f])
                assert res.tracked == 1 and dt < 0.005 and dr < 0.3, (f, dt, dr)
                tracked.append(f)
    assert tracked == [15, 25]


def median_scene_error(rec, st, f):
    pose64 = torch.from_numpy(S.trajectory(st.frame_count)[f]).to("cuda")
    gt, _ = S._raycast(VGA, pose64, "cuda")
    out = rec.render(st.frame_T_global[f], VGA.width, VGA.height, VGA.fx, VGA.fy, VGA.cx, VGA.cy, near=0.1,
                     far=20.0, outputs=("depth",))
    depth = out["depth"].double()
    both = torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0) & (depth > 0)
    return float(np.median((depth - gt)[both].abs().cpu().numpy()))


# A 120-frame VGA stream tracked from frame 0's pose alone: the largest error against the ground-truth trajectory,
# and the final cloud's median depth error against the ray-cast scene relative to the same stream integrated with
# the ground-truth poses.
@pytest.mark.parametrize("sigma,max_t,max_r", [(None, 0.01, 0.5), (0.0, 0.002, 0.1)], ids=["nominal_noise", "noise_free"])
def test_pose_free_stream(sigma, max_t, max_r):
    st = S.make_stream(VGA, 120, sigma_depth=sigma, device="cuda")
    pp, ip = params(VGA)
    rec = make()
    with R.TrackedSession(rec, pp, ip, st.global_T_frame[0]) as s:
        for f in range(st.frame_count):
            s.push(st.depth[f], st.color[f])
    errors = np.array([pose_error(s.trajectory[f], st.global_T_frame[f]) for f in range(st.frame_count)])
    lost = sum(1 for r in s.results if not r.tracked)
    reference = make()
    first, last = st.integrated_range()
    reference.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                         ip, first, last)
    f = last - 4
    tracked_error, reference_error = median_scene_error(rec, st, f), median_scene_error(reference, st, f)
    print(f"pose-free sigma={sigma}: max {errors[:, 0].max() * 1000:.3f} mm / {errors[:, 1].max():.4f} deg, "
          f"mean {errors[:, 0].mean() * 1000:.3f} mm / {errors[:, 1].mean():.4f} deg, lost {lost}; "
          f"median scene error {tracked_error * 1000:.3f} mm vs {reference_error * 1000:.3f} mm with true poses")
    assert errors[:, 0].max() <= max_t and errors[:, 1].max() <= max_r
    assert tracked_error <= 1.5 * reference_error
