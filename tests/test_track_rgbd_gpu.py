"""sm_track_frame_rgbd / sm_track_linearize_rgbd on the GPU: the joint linearisation against the numpy restatement
(tests/track_rgbd_walk.py), weight 0 against sm_track_frame, pose recovery on exact data and on a single textured wall
that depth alone cannot track, pose-free wall and desk streams (TrackedSession with rgbd), determinism, read-only
behaviour, lost frames and argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import TrackParams, TrackRGBDParams, TrackRGBDResult
from tests import track_rgbd_walk as RW
from tests import track_walk as TW
from tests.util import offset, params

pytestmark = pytest.mark.gpu

VGA = S.Camera.tum(640, 480)
QVGA = S.Camera.tum(320, 240)
SMALL = S.Camera.tum(160, 120)
CAP = 2_000_000
SCALE = 5000.0
pose_error = TW.pose_error


def cam_tuple(cam):
    return (cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


def make(cam=VGA):
    return R.CUDASurfelReconstruction(CAP, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


def cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t.to(dtype) if dtype is not None else t).cuda()


def u16(a):
    return cuda(np.asarray(a).astype(np.int32), torch.uint16)


def assert_parity(rec, level, live, live_color, model_depth, model_normal, model_color, T, cam):
    rp = TrackRGBDParams.defaults()
    lc = TW.scaled(cam_tuple(cam), level)
    system, rc2, inliers, photo = rec.track_linearize_rgbd(level, u16(live), cuda(live_color), cuda(model_depth),
                                                           cuda(model_normal), cuda(model_color), T, rgbd=rp)
    live_I = RW.pyramid(RW.intensity(live_color), cam_tuple(cam), level + 1)[level]
    model_I = RW.pyramid(RW.model_intensity(model_color, model_depth), cam_tuple(cam), level + 1)[level]
    ref = RW.linearize(live, SCALE, lc[2:], model_depth, model_normal, cam_tuple(cam)[2:], np.asarray(T, np.float32),
                       live_I, model_I, rp.photometric_weight, rp.max_intensity_residual, rp.min_gradient)
    assert (inliers, photo) == (ref["inliers"], ref["photometric_inliers"])
    assert photo > 0
    bound = 1e-9 * ref["magnitude"] + 1e-300
    bad = np.abs(system - ref["system"]) > bound
    assert not bad.any(), (np.flatnonzero(bad), system[bad], ref["system"][bad])
    rc_terms = ref["rc"].astype(np.float64) ** 2
    assert abs(rc2 - ref["rc2"]) <= 1e-9 * rc_terms.sum() + 1e-300


OFFSETS = {"identity": ((0, 0, 0), (0, 0, 0)), "small": ((0.3, -0.2, 0.4), (0.005, -0.004, 0.006)),
           "large": ((1.5, 1.0, -2.0), (0.02, 0.03, -0.025))}


@pytest.mark.parametrize("scene", sorted(TW.SCENES))
@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("off", sorted(OFFSETS))
def test_linearize_rgbd_matches_restatement_on_textured_planes(scene, level, off):
    cam = cam_tuple(SMALL)
    z, n, color = RW.render_textured_planes(TW.SCENES[scene], cam, np.eye(4)[:3])
    model_depth = np.where(np.isfinite(z), z, 0).astype(np.float32)
    model_normal = n.astype(np.float32)
    model_depth[10:14, 20:30] = np.nan
    model_depth[40:44, 50:58] = 0
    model_normal[60:62, 60:70] = np.nan
    truth = offset((0.5, -0.8, 0.3), (0.01, 0.005, -0.01))
    zl, _, _ = RW.render_textured_planes(TW.SCENES[scene], TW.scaled(cam, level), truth)
    _, _, live_color = RW.render_textured_planes(TW.SCENES[scene], cam, truth)
    live = TW.quantize(zl)
    live[3:6, 3:12] = 0
    rec = make(SMALL)
    assert_parity(rec, level, live, live_color, model_depth, model_normal, color,
                  offset(*OFFSETS[off]).astype(np.float32), SMALL)


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


def model_view(rec, global_T_camera, cam=VGA):
    out = rec.render(R.invert_rigid(global_T_camera), cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy,
                     near=0.1, far=100.0, outputs=("depth", "normal", "color"))
    torch.cuda.synchronize()
    return out["depth"].cpu().numpy(), out["normal"].cpu().numpy(), out["color"].cpu().numpy()


@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("off", sorted(OFFSETS))
def test_linearize_rgbd_matches_restatement_on_a_rendered_cloud(integrated, level, off):
    st, rec = integrated
    model_depth, model_normal, model_color = model_view(rec, st.global_T_frame[30])
    raw = st.depth[31].cuda()
    lc = TW.scaled(cam_tuple(VGA), level)
    live = R.DownscaleUsingMedianWhileExcluding(None, 0, lc[0], lc[1], raw).cpu().numpy() if level else raw.cpu().numpy()
    rel = TW.compose(R.invert_rigid(st.global_T_frame[30]), st.global_T_frame[31])
    T = TW.compose(offset(*OFFSETS[off]), rel).astype(np.float32)
    assert_parity(rec, level, live, st.color[31].cpu().numpy(), model_depth, model_normal, model_color, T, VGA)


def test_weight_zero_is_sm_track_frame(integrated):
    st, rec = integrated
    pp, _ = params(VGA)
    rp = TrackRGBDParams.defaults()
    rp.photometric_weight = 0.0
    depth, color = st.depth[32].cuda(), st.color[32].cuda()
    guess = TW.compose(st.global_T_frame[32], offset((0.5, 0.5, 0), (0.01, 0, 0))).astype(np.float32)
    seed = (st.depth[31].cuda(), st.color[31].cuda(), st.global_T_frame[31])
    for source in ("cloud", "previous"):
        # the previous frame of each call: frame 31 tracked by the same kind of call
        rec.track(seed[0], seed[2], pp=pp)
        a, ra = rec.track(depth, guess, pp=pp, source=source)
        rec.track_rgbd(*seed, rgbd=rp, pp=pp)
        b, rb = rec.track_rgbd(depth, color, guess, rgbd=rp, pp=pp, source=source)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), source
        assert bytes(ra) == bytes(rb.depth), source
        assert rb.photometric_inliers == 0 and rb.rms_intensity == 0.0
        assert ra.tracked == 1


def quantized_render(rec, global_T_camera, cam=VGA):
    depth, _, color = model_view(rec, global_T_camera, cam)
    return u16(TW.quantize(depth.astype(np.float64), SCALE)), cuda(color)


@pytest.mark.parametrize("perturbation", [((1.2, -1.1, 1.15), (0.012, -0.011, 0.0115)), ((0, 0, 0), (0.03, -0.03, 0.026)),
                                          ((0, 0, 5.0), (0, 0, 0))], ids=["2cm_2deg", "5cm", "5deg_roll"])
def test_recovers_the_pose_of_exact_data(integrated, perturbation):
    st, rec = integrated
    pose = st.global_T_frame[30]
    live, color = quantized_render(rec, pose)
    guess = TW.compose(pose, offset(*perturbation)).astype(np.float32)
    pp, _ = params(VGA)
    out, res = rec.track_rgbd(live, color, guess, pp=pp)
    dt, dr = pose_error(out, pose)
    print(f"exact data rgbd: {dt * 1000:.3f} mm, {dr:.4f} deg, {res.depth.iterations} steps, photometric inliers "
          f"{res.photometric_inliers}, rms {res.rms_intensity:.2f}")
    assert res.depth.tracked == 1
    assert dt <= 1e-3 and dr <= 0.05


def wall_stream(cam, frames):
    depth, color, poses = RW.wall_stream(cam_tuple(cam), frames)
    g = poses.astype(np.float32)
    return (torch.from_numpy(depth.astype(np.int32)).to(torch.uint16).cuda(), torch.from_numpy(color).cuda(), g,
            S.invert_poses(poses).astype(np.float32), S.others_TR_reference(poses, SCALE, 8))


@pytest.fixture(scope="module")
def wall():
    return wall_stream(QVGA, 90)


def test_single_textured_plane_needs_colour(wall):
    depth, color, g, f, others = wall
    pp, ip = params(QVGA)
    rec = make(QVGA)
    rec.stream_run(None, depth[:40], color[:40], g[:40], f[:40], others[:40], pp, ip, 4, 36)
    torch.cuda.synchronize()
    pose = g[34]
    n = np.array([0.0, 0.0, 1.0])   # the wall's normal in the world
    slide = np.concatenate([Rotation.from_rotvec(np.radians(1.0) * n).as_matrix(), np.array([[0.01], [-0.006], [0.0]])],
                           axis=1)
    guess = TW.compose(slide, pose).astype(np.float32)
    out, res = rec.track_rgbd(depth[34], color[34], guess, pp=pp)
    dt, dr = pose_error(out, pose)
    out0, res0 = rec.track(depth[34], guess, pp=pp)
    dt0, dr0 = pose_error(out0, pose)
    print(f"wall, guess {pose_error(guess, pose)}: rgbd {dt * 1000:.3f} mm / {dr:.4f} deg; depth only tracked "
          f"{res0.tracked}: {dt0 * 1000:.3f} mm / {dr0:.4f} deg")
    # measured on an H100: RGB-D 0.59 mm / 0.04 deg, depth only 3.5 mm / 0.17 deg from a 9 mm + 1 deg in-plane guess
    assert res.depth.tracked == 1 and dt <= 1.5e-3 and dr <= 0.1
    assert res0.tracked == 0 or dt0 >= 2.5e-3 or dr0 >= 0.15


def pose_free(cam, depth, color, first_pose, rgbd, frames):
    pp, ip = params(cam)
    rec = make(cam)
    with R.TrackedSession(rec, pp, ip, first_pose, rgbd=rgbd) as s:
        for k in range(frames):
            s.push(depth[k], color[k])
    return rec, s


def test_pose_free_wall_stream(wall):
    depth, color, g, _, _ = wall
    _, s = pose_free(QVGA, depth, color, g[0], TrackRGBDParams.defaults(), 90)
    _, s0 = pose_free(QVGA, depth, color, g[0], None, 90)
    e = np.array([pose_error(s.trajectory[k], g[k]) for k in range(90)])
    e0 = np.array([pose_error(s0.trajectory[k], g[k]) for k in range(90)])
    lost = sum(1 for r in s.results if not r.depth.tracked)
    print(f"pose-free wall: rgbd max {e[:, 0].max() * 1000:.3f} mm / {e[:, 1].max():.4f} deg, lost {lost}; depth only "
          f"max {e0[:, 0].max() * 1000:.3f} mm / {e0[:, 1].max():.4f} deg, lost "
          f"{sum(1 for r in s0.results if not r.tracked)}")
    # measured on an H100: RGB-D 2.9 mm / 0.22 deg; depth only drifts by more than half a metre
    assert e[:, 0].max() <= 0.006 and e[:, 1].max() <= 0.5
    assert e0[:, 0].max() > 2 * e[:, 0].max()


@pytest.mark.parametrize("sigma,max_t,max_r", [(None, 0.01, 0.5), (0.0, 0.002, 0.1)], ids=["nominal_noise", "noise_free"])
def test_pose_free_desk_stream(sigma, max_t, max_r):
    st = S.make_stream(VGA, 120, sigma_depth=sigma, device="cuda")
    _, s = pose_free(VGA, st.depth, st.color, st.global_T_frame[0], TrackRGBDParams.defaults(), 120)
    e = np.array([pose_error(s.trajectory[f], st.global_T_frame[f]) for f in range(120)])
    lost = sum(1 for r in s.results if not r.depth.tracked)
    print(f"pose-free desk rgbd sigma={sigma}: max {e[:, 0].max() * 1000:.3f} mm / {e[:, 1].max():.4f} deg, mean "
          f"{e[:, 0].mean() * 1000:.3f} mm / {e[:, 1].mean():.4f} deg, lost {lost}")
    assert e[:, 0].max() <= max_t and e[:, 1].max() <= max_r


def test_two_calls_are_bit_identical_and_read_only(integrated):
    st, rec = integrated
    pp, _ = params(VGA)
    before, n0, m0 = rec.dump_state()
    before = before.copy()
    guess = TW.compose(st.global_T_frame[32], offset((0.5, 0.5, 0), (0.01, 0, 0))).astype(np.float32)
    a, ra = rec.track_rgbd(st.depth[32].cuda(), st.color[32].cuda(), guess, pp=pp)
    b, rb = rec.track_rgbd(st.depth[32].cuda(), st.color[32].cuda(), guess, pp=pp)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and bytes(ra) == bytes(rb)
    assert ra.depth.tracked == 1 and ra.photometric_inliers > 0
    rec.track_rgbd(st.depth[33].cuda(), st.color[33].cuda(), st.global_T_frame[33], pp=pp, source="previous")
    after, n1, m1 = rec.dump_state()
    assert (n0, m0) == (n1, m1)
    assert np.array_equal(before.view(np.uint32), after.view(np.uint32))


def test_lost_frames_return_the_guess(integrated):
    st, rec = integrated
    pp, _ = params(VGA)
    guess = st.global_T_frame[20]
    out, res = make().track_rgbd(st.depth[20].cuda(), st.color[20].cuda(), guess, pp=pp)
    assert res.depth.tracked == 0 and np.array_equal(out, np.asarray(guess, np.float32))
    assert res.photometric_inliers == 0
    far = TW.compose(st.global_T_frame[20], offset((0, 0, 0), (0.0, 0.0, 1.0))).astype(np.float32)
    out, res = rec.track_rgbd(st.depth[20].cuda(), st.color[20].cuda(), far, pp=pp)
    assert res.depth.tracked == 0 and np.array_equal(out, far)


def test_invalid_arguments_are_rejected_without_a_launch(product):
    rec = make(SMALL)
    pp, _ = params(SMALL)
    W, H = SMALL.width, SMALL.height
    depth = torch.zeros((H, W), dtype=torch.uint16, device="cuda")
    color = torch.zeros((H, W, 3), dtype=torch.uint8, device="cuda")
    md = torch.zeros((H, W), dtype=torch.float32, device="cuda")
    mn = torch.zeros((H, W, 3), dtype=torch.float32, device="cuda")
    I = np.eye(4, dtype=np.float32)[:3].copy()
    out = np.zeros(12, np.float32)
    sysv = np.zeros(27, np.float64)
    rc2, inl, photo = C.c_double(), C.c_uint32(), C.c_uint32()
    fn = rec.lib.fn

    def frame(tp=None, rp=True, cptr=color.data_ptr(), cpitch=3 * W, guess=I, rgbd=None):
        tp = tp or TrackParams.defaults()
        r = TrackRGBDResult()
        rp = (rgbd or TrackRGBDParams.defaults()) if rp else None
        return fn["track_frame_rgbd"](rec._h, None, C.byref(tp), C.byref(pp), C.byref(rp) if rp else None,
                                      depth.data_ptr(), 2 * W, cptr, cpitch, guess.ctypes.data_as(C.c_void_p),
                                      out.ctypes.data_as(C.c_void_p), C.byref(r))

    def lin(level=0, rp=True, live_color=color.data_ptr(), live_color_pitch=3 * W, model_color=color.data_ptr(),
            model_color_pitch=3 * W, rgbd=None):
        tp = TrackParams.defaults()
        rp = (rgbd or TrackRGBDParams.defaults()) if rp else None
        return fn["track_linearize_rgbd"](rec._h, None, C.byref(tp), C.byref(rp) if rp else None, level, SCALE,
                                          depth.data_ptr(), 2 * W, live_color, live_color_pitch, md.data_ptr(), 4 * W,
                                          mn.data_ptr(), 12 * W, model_color, model_color_pitch,
                                          I.ctypes.data_as(C.c_void_p), sysv.ctypes.data_as(C.c_void_p),
                                          C.byref(rc2), C.byref(inl), C.byref(photo))

    def rgbd_with(**kw):
        rp = TrackRGBDParams.defaults()
        for k, v in kw.items():
            setattr(rp, k, v)
        return rp

    torch.cuda.synchronize()
    launches = product.fn["kernel_launch_count"]()
    bad = _lib.SM_ERR_INVALID_ARGUMENT
    nan, inf = float("nan"), float("inf")
    prev = TrackParams.defaults()
    prev.model_source = _lib.TRACK_PREVIOUS_FRAME
    assert frame(prev) == bad
    assert frame(rp=False) == bad and frame(cptr=None) == bad and frame(cpitch=3 * W - 1) == bad
    for field in ("photometric_weight", "max_intensity_residual", "min_gradient"):
        for value in (nan, inf, -1.0):
            assert frame(rgbd=rgbd_with(**{field: value})) == bad, (field, value)
            assert lin(rgbd=rgbd_with(**{field: value})) == bad, (field, value)
    levels0 = TrackParams.defaults()
    levels0.levels = 0
    assert frame(levels0) == bad
    assert lin(rp=False) == bad and lin(live_color=None) == bad and lin(model_color=None) == bad
    assert lin(live_color_pitch=3 * W - 1) == bad and lin(model_color_pitch=3 * W - 1) == bad and lin(level=4) == bad
    with pytest.raises(ValueError):
        rec.track_rgbd(depth, color[:, :-1], I)
    torch.cuda.synchronize()
    assert product.fn["kernel_launch_count"]() == launches
    # a depth-only call in between leaves no kept intensity for the previous-frame source
    assert frame() == _lib.SM_OK
    assert frame(prev) == _lib.SM_OK
    rec.track(depth, I, pp=pp)
    torch.cuda.synchronize()
    launches = product.fn["kernel_launch_count"]()
    assert frame(prev) == bad
    assert product.fn["kernel_launch_count"]() == launches
    assert lin(level=1) == _lib.SM_OK and frame() == _lib.SM_OK and frame(prev) == _lib.SM_OK


def test_launch_count_does_not_depend_on_the_data(integrated, product):
    st, rec = integrated
    pp, _ = params(VGA)
    counts = []
    for guess in (st.global_T_frame[32], TW.compose(st.global_T_frame[32], offset((0, 0, 0), (0, 0, 1.0)))):
        torch.cuda.synchronize()
        before = product.fn["kernel_launch_count"]()
        rec.track_rgbd(st.depth[32].cuda(), st.color[32].cuda(), np.asarray(guess, np.float32), pp=pp)
        counts.append(product.fn["kernel_launch_count"]() - before)
    assert counts[0] == counts[1]
