"""The tracking rules without a GPU: the numpy restatement (tests/track_walk.py) against finite differences, scipy's
rotation vector and a Gauss-Newton loop on analytic plane scenes; the ctypes layout and defaults of sm_track_*."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from surfelmeshing_b200 import _lib
from tests import track_walk as TW

CAM = (160, 120, 131.25, 131.25, 80.0, 60.0)   # TUM fr1 intrinsics at 160 x 120, pixel-corner convention


def offset(rotvec_deg, translation):
    R = Rotation.from_rotvec(np.radians(rotvec_deg)).as_matrix()
    return np.concatenate([R, np.asarray(translation, float)[:, None]], axis=1)


def scene_images(name, model_T_live, level=0, holes=False):
    """Model images from the identity camera and the live u16 image from model_T_live, both of the plane scene."""
    z, n = TW.render_planes(TW.SCENES[name], CAM, np.eye(4)[:3])
    model_depth = np.where(np.isfinite(z), z, 0).astype(np.float32)
    model_normal = n.astype(np.float32)
    live_cam = TW.scaled(CAM, level)
    zl, _ = TW.render_planes(TW.SCENES[name], live_cam, model_T_live)
    live = TW.quantize(zl)
    if holes:
        model_depth[10:14, 20:30] = np.nan
        model_depth[40:44, 50:58] = 0
        live[5:9, 5:20] = 0
    return live, live_cam, model_depth, model_normal


def test_jacobian_matches_finite_differences():
    T = offset((0.5, -1.0, 0.7), (0.01, -0.02, 0.015)).astype(np.float32)
    live, lc, md, mn = scene_images("corner", T)
    lin = TW.linearize(live, 5000.0, lc[2:], md, mn, CAM[2:], T)
    assert lin["inliers"] > 1000
    rng = np.random.RandomState(1)
    h = 1e-6
    for k in rng.choice(lin["inliers"], 50, replace=False):
        p, q, n = (lin[key][k].astype(np.float64) for key in ("p", "q", "n"))
        fd = np.zeros(6)
        for j in range(6):
            step = np.zeros(6)
            step[j] = h
            plus = TW.residual(p, TW.compose(TW.se3_exp(step), T), n, q)
            minus = TW.residual(p, TW.compose(TW.se3_exp(-step), T), n, q)
            fd[j] = (plus - minus) / (2 * h)
        J = lin["J"][k].astype(np.float64)
        assert np.abs(J - fd).max() <= 1e-6 * max(np.abs(fd).max(), 1.0), (k, J, fd)


@pytest.mark.parametrize("rotvec", [(0, 0, 0), (1e-6, -2e-6, 3e-6), (1e-4, 0, 0), (0.01, -0.02, 0.03), (0.5, 1.0, -0.3),
                                    (2.0, -1.0, 0.5)])
def test_se3_exponential_rotation_matches_scipy(rotvec):
    xi = np.concatenate([rotvec, [0.1, -0.2, 0.3]])
    T = TW.se3_exp(xi)
    assert np.abs(T[:, :3] - Rotation.from_rotvec(rotvec).as_matrix()).max() <= 1e-12
    # the translation is V v; exp of a pure translation is the translation itself
    assert np.allclose(TW.se3_exp(np.array([0, 0, 0, 0.1, -0.2, 0.3]))[:, 3], [0.1, -0.2, 0.3], atol=0)


@pytest.mark.parametrize("scene", ["corner"])
@pytest.mark.parametrize("level", [0, 1])
def test_gauss_newton_on_the_restatement_converges(scene, level):
    truth = offset((1.0, -1.5, 0.8), (0.02, -0.015, 0.01)).astype(np.float32)
    live, lc, md, mn = scene_images(scene, truth, level, holes=True)
    T = TW.gauss_newton(live, 5000.0, lc[2:], md, mn, CAM[2:], np.eye(4)[:3], iterations=12)
    dt = np.abs(T[:, 3].astype(np.float64) - truth[:, 3]).max()
    R = T[:, :3].astype(np.float64) @ truth[:, :3].astype(np.float64).T
    angle = math.degrees(math.acos(min(1.0, (np.trace(R) - 1) / 2)))
    assert dt < 1e-3 and angle < 0.05, (dt, angle)


def test_restatement_rules_on_holes_and_gates():
    """Holes in the live image remove pixels from the valid count; NaN and zero model depths are never inliers; a
    live frame far off has no inliers."""
    T = np.eye(4, dtype=np.float32)[:3]
    live, lc, md, mn = scene_images("fronto_parallel", T, holes=True)
    lin = TW.linearize(live, 5000.0, lc[2:], md, mn, CAM[2:], T)
    interior = (CAM[0] - 2) * (CAM[1] - 2)
    assert lin["valid"] < interior and lin["inliers"] < lin["valid"]
    far = offset((0, 0, 0), (0, 0, 1.0)).astype(np.float32)
    assert TW.linearize(live, 5000.0, lc[2:], md, mn, CAM[2:], far)["inliers"] == 0


def test_track_struct_layouts():
    assert C.sizeof(_lib.TrackParams) == 44
    assert C.sizeof(_lib.TrackResult) == 20
    assert [f for f, _ in _lib.TrackParams._fields_] == [
        "levels", "iterations", "max_point_distance", "max_normal_angle_deg", "min_inlier_fraction",
        "convergence_rotation", "convergence_translation", "model_source"]


def test_default_track_params_match(product):
    tp = _lib.TrackParams()
    product.fn["default_track_params"](C.byref(tp))
    d = _lib.TrackParams.defaults()
    for name, _ in tp._fields_:
        a, b = getattr(tp, name), getattr(d, name)
        if name == "iterations":
            a, b = list(a), list(b)
        assert a == b, name
    assert list(tp.iterations) == [4, 5, 10, 0] and tp.levels == 3 and tp.model_source == _lib.TRACK_CLOUD


def test_pose_chain_stays_rigid():
    """Frame-to-frame tracking of a noise-free 160 x 120 stream with sm_track_frame's pose bookkeeping. With the
    nearest-rotation projection the error grows about linearly (resolution-limited drift); without it the fp32 poses
    leave SO(3), the transpose-as-inverse and the left-multiplied update amplify the scale error every frame, and
    the chain falls apart within a few frames."""
    from surfelmeshing_b200 import synthetic as S
    cam = S.Camera.tum(160, 120)
    ct = (cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    st = S.make_stream(cam, 14, sigma_depth=0.0, dropout=0.0)
    depths = [np.where(st.depth[k].numpy() < 15000, st.depth[k].numpy(), 0).astype(np.uint16) for k in range(14)]
    traj = TW.track_previous_frame_chain(depths, st.global_T_frame[0], ct)
    errors = np.array([TW.pose_error(traj[k], st.global_T_frame[k]) for k in range(14)])
    assert errors[:, 0].max() <= 0.01 and errors[:, 1].max() <= 0.5, errors
    for k in range(1, 14):
        assert abs(np.linalg.det(traj[k][:, :3].astype(np.float64)) - 1) < 1e-6
    with np.errstate(all="ignore"):
        try:
            bad = TW.track_previous_frame_chain(depths, st.global_T_frame[0], ct, project=False)
            drifted = max(TW.pose_error(bad[k], st.global_T_frame[k])[0] for k in range(14))
        except np.linalg.LinAlgError:
            drifted = math.inf
    assert drifted > 10 * errors[:, 0].max()


def test_five_degree_guesses_inlier_fraction():
    """Why a 5-degree tilt is reported lost and a 5-degree roll is not: the correspondence gate is the point-to-point
    distance |p - q| <= 5 cm at the pixel a live point projects to. Turning the model camera by 5 degrees about an
    axis across the view moves every pixel's ray ~5 degrees, which at 1-3 m puts ~9-26 cm between p and q almost
    everywhere; a roll about the optical axis moves the rays near the image centre little. Measured with the
    restatement on frame 30 of the VGA synthetic stream (ray-cast, cut at the 3 m max_depth), before the first step
    (T = identity): the tilt keeps well under min_inlier_fraction = 0.1 of the valid pixels, the roll far more."""
    import torch
    from surfelmeshing_b200 import synthetic as S
    cam = S.Camera.tum(640, 480)
    ct = (cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    pose = S.trajectory(31)[30]

    def image(global_T_camera):
        z, _ = S._raycast(cam, torch.from_numpy(np.asarray(global_T_camera, np.float64)), "cpu")
        z = z.numpy()
        return TW.quantize(np.where(z < 3.0, z, np.inf))

    live = image(pose)
    fractions = {}
    for name, rotvec in (("tilt", 5.0 * np.array([3.0, -2.6, 2.9]) / np.linalg.norm([3.0, -2.6, 2.9])),
                         ("roll", (0.0, 0.0, 5.0))):
        guess = TW.compose(pose, offset(rotvec, (0, 0, 0)))
        md, mn = TW.live_view(image(guess), 5000.0, ct)
        lin = TW.linearize(live, 5000.0, ct[2:], md, mn, ct[2:], np.eye(4, dtype=np.float32)[:3])
        fractions[name] = lin["inliers"] / lin["valid"]
    print(fractions)
    assert fractions["tilt"] < 0.1 < fractions["roll"]
