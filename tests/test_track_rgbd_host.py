"""The RGB-D tracking rules without a GPU: the numpy restatement (tests/track_rgbd_walk.py) against finite differences,
the pyramid's edge rule, the rank of the depth-only and the joint systems on a single textured plane, Gauss-Newton on
the restatement, weight 0, and the ctypes layout and defaults of sm_track_rgbd_*."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from surfelmeshing_b200 import _lib
from tests import track_rgbd_walk as RW
from tests import track_walk as TW

CAM = (160, 120, 131.25, 131.25, 80.0, 60.0)   # TUM fr1 intrinsics at 160 x 120, pixel-corner convention
WEIGHTS = dict(photometric_weight=2e-4, max_intensity_residual=40.0, min_gradient=2.0)


def offset(rotvec_deg, translation):
    R = Rotation.from_rotvec(np.radians(rotvec_deg)).as_matrix()
    return np.concatenate([R, np.asarray(translation, float)[:, None]], axis=1)


def textured_images(name, model_T_live, level=0):
    """Model depth, normal and intensity from the identity camera, the live u16 level image and the live intensity
    pyramid from model_T_live, of the textured plane scene."""
    z, n, c = RW.render_textured_planes(TW.SCENES[name], CAM, np.eye(4)[:3])
    model_depth = np.where(np.isfinite(z), z, 0).astype(np.float32)
    zl, _, cl = RW.render_textured_planes(TW.SCENES[name], TW.scaled(CAM, level), model_T_live)
    _, _, cl0 = RW.render_textured_planes(TW.SCENES[name], CAM, model_T_live)
    live_I = RW.pyramid(RW.intensity(cl0), CAM, level + 1)
    model_I = RW.pyramid(RW.model_intensity(c, model_depth), CAM, level + 1)
    return TW.quantize(zl), model_depth, n.astype(np.float32), live_I, model_I


def in_plane_offset(name, angle_deg, shift):
    """A pose turned by angle_deg about the plane's normal and shifted by `shift` metres along the plane."""
    n = np.asarray(TW.SCENES[name][0][0])
    u, _ = RW.tangent_basis(n)
    return np.concatenate([Rotation.from_rotvec(np.radians(angle_deg) * n).as_matrix(), (shift * u)[:, None]], axis=1)


def test_photometric_jacobian_matches_finite_differences():
    T = offset((0.5, -1.0, 0.7), (0.01, -0.02, 0.015)).astype(np.float32)
    live, md, mn, live_I, model_I = textured_images("corner", T)
    lin = RW.linearize(live, 5000.0, CAM[2:], md, mn, CAM[2:], T, live_I[0], model_I[0], **WEIGHTS)
    assert lin["photometric_inliers"] > 1000
    rng = np.random.RandomState(2)
    h = 1e-6
    checked = 0
    for k in rng.permutation(lin["photometric_inliers"]):
        p, i, j = lin["p"][k].astype(np.float64), int(lin["i"][k]), int(lin["j"][k])
        # inside the bilinear cell, away from its edges, so the central differences stay in it
        pm = T[:, :3].astype(np.float64) @ p + T[:, 3]
        a = CAM[2] * pm[0] / pm[2] + CAM[4] - 0.5 - i
        b = CAM[3] * pm[1] / pm[2] + CAM[5] - 0.5 - j
        if not (0.05 < a < 0.95 and 0.05 < b < 0.95):
            continue
        live_value = float(live_I[0][lin["y"][k], lin["x"][k]])
        fd = np.zeros(6)
        for m in range(6):
            step = np.zeros(6)
            step[m] = h
            plus = RW.photometric_residual(p, TW.compose(TW.se3_exp(step), T), model_I[0], CAM[2:], i, j, live_value)
            minus = RW.photometric_residual(p, TW.compose(TW.se3_exp(-step), T), model_I[0], CAM[2:], i, j, live_value)
            fd[m] = (plus - minus) / (2 * h)
        J = lin["Jc"][k].astype(np.float64)
        assert np.abs(J - fd).max() <= 1e-4 * max(np.abs(fd).max(), 1.0), (k, J, fd)
        checked += 1
        if checked == 50:
            break
    assert checked == 50


@pytest.mark.parametrize("size", [(160, 120), (161, 121), (97, 73), (100, 75), (33, 17), (641, 479), (1279, 959)])
def test_pyramid_indices_stay_inside_odd_and_uneven_sizes(size):
    """P2 at the sizes Camera.scaled produces: 2x and 2y never pass the edge (downscale asserts it), the clamped
    neighbour is taken only at the last column / row of an odd size, and a NaN child makes its parent NaN."""
    w, h = size
    cam = (w, h, 0.8 * w, 0.8 * w, w / 2, h / 2)
    rng = np.random.RandomState(w * 1000 + h)
    I0 = RW.intensity(rng.randint(0, 256, (h, w, 3)).astype(np.uint8))
    I0[h // 2, w // 3] = np.nan
    levels = RW.pyramid(I0, cam, 4)
    for l in range(1, 4):
        lw, lh = TW.scaled(cam, l)[:2]
        assert levels[l].shape == (lh, lw)
        src = levels[l - 1]
        # a direct restatement of one pixel in the last row and column
        x, y = lw - 1, lh - 1
        x1, y1 = min(2 * x + 1, src.shape[1] - 1), min(2 * y + 1, src.shape[0] - 1)
        want = ((src[2 * y, 2 * x] + src[2 * y, x1]) + (src[y1, 2 * x] + src[y1, x1])) * np.float32(0.25)
        assert np.array_equal(levels[l][y, x], want, equal_nan=True)
    assert np.isnan(levels[1][(h // 2) // 2, (w // 3) // 2])


def test_single_plane_leaves_the_depth_system_rank_three():
    """On the textured fronto-parallel plane the depth-only J^T J has three eigenvalues at rounding level (sliding
    along the plane and turning about its normal are free); the joint system is well conditioned."""
    T = np.eye(4, dtype=np.float32)[:3]
    live, md, mn, live_I, model_I = textured_images("fronto_parallel", T)
    lin = RW.linearize(live, 5000.0, CAM[2:], md, mn, CAM[2:], T, live_I[0], model_I[0], **WEIGHTS)
    depth = np.linalg.eigvalsh(TW.unpack(lin["depth_system"])[0])
    joint = np.linalg.eigvalsh(TW.unpack(lin["system"])[0])
    print("depth-only", depth / depth.max(), "joint", joint / joint.max())
    assert np.all(np.abs(depth[:3]) <= 1e-12 * depth.max())
    assert joint.min() >= 1e-3 * joint.max()


@pytest.mark.parametrize("scene", ["tilted", "fronto_parallel"])
def test_gauss_newton_recovers_an_in_plane_offset_only_with_colour(scene):
    truth = in_plane_offset(scene, 1.0, 0.01).astype(np.float32)
    live, md, mn, live_I, model_I = textured_images(scene, truth)
    start = np.eye(4, dtype=np.float32)[:3]
    T = RW.gauss_newton(live, 5000.0, CAM[2:], md, mn, CAM[2:], start, live_I[0], model_I[0], iterations=15,
                        photometric_weight=2e-4)
    dt, dr = TW.pose_error(T, truth)
    assert dt < 1.2e-3 and dr < 0.02, (dt, dr)
    # the depth-only system is singular: no step, or a step of arbitrary size in its null space
    try:
        T0 = RW.gauss_newton(live, 5000.0, CAM[2:], md, mn, CAM[2:], start, live_I[0], model_I[0], iterations=15,
                             photometric_weight=0.0)
        dt0, dr0 = TW.pose_error(T0, truth)
    except np.linalg.LinAlgError:
        dt0, dr0 = np.inf, np.inf
    assert dt0 > 5e-3 or dr0 > 0.5, (dt0, dr0)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_weight_zero_is_the_depth_system(level):
    T = offset((0.5, -0.8, 0.3), (0.01, 0.005, -0.01)).astype(np.float32)
    live, md, mn, live_I, model_I = textured_images("corner", T, level)
    lc = TW.scaled(CAM, level)
    lin = RW.linearize(live, 5000.0, lc[2:], md, mn, CAM[2:], T, live_I[level], model_I[level], 0.0, 40.0, 2.0)
    ref = TW.linearize(live, 5000.0, lc[2:], md, mn, CAM[2:], T)
    assert np.array_equal(lin["system"], ref["system"])
    assert lin["inliers"] == ref["inliers"] and lin["photometric_inliers"] > 0


def test_track_rgbd_struct_layouts():
    assert C.sizeof(_lib.TrackRGBDParams) == 12
    assert C.sizeof(_lib.TrackRGBDResult) == 28
    assert [f for f, _ in _lib.TrackRGBDParams._fields_] == ["photometric_weight", "max_intensity_residual",
                                                             "min_gradient"]
    assert [f for f, _ in _lib.TrackRGBDResult._fields_] == ["depth", "photometric_inliers", "rms_intensity"]
    assert _lib.TrackRGBDResult.photometric_inliers.offset == 20


def test_default_track_rgbd_params_match(product):
    rp = _lib.TrackRGBDParams()
    product.fn["default_track_rgbd_params"](C.byref(rp))
    d = _lib.TrackRGBDParams.defaults()
    for name, _ in rp._fields_:
        assert getattr(rp, name) == getattr(d, name), name
