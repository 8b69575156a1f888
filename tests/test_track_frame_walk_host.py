"""The frame walk of tests/track_walk.py without a GPU: its solve, SE(3) increment and polar projection against plain
float64 references (numpy, scipy), its loss and clear rules on constructed edges, and the whole coarse-to-fine
schedule on the analytic plane scenes with the restated linearisation in place of the device's."""
import math

import numpy as np
import pytest
from scipy.linalg import expm
from scipy.spatial.transform import Rotation

from surfelmeshing_b200._lib import TrackParams
from tests import track_walk as TW
from tests.util import offset

CAM = (160, 120, 131.25, 131.25, 80.0, 60.0)   # TUM fr1 intrinsics at 160 x 120, pixel-corner convention
EPS = np.finfo(np.float64).eps


def pack(A, g):
    """The 27 sums of a system J^T J = A, J^T r = g."""
    return np.array([A[i, j] for i in range(6) for j in range(i, 6)] + list(g), np.float64)


# ---- the solve -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cond", [1.0, 1e3, 1e6, 1e8, 1e10])
def test_cholesky_solve_matches_numpy(cond):
    rng = np.random.RandomState(int(math.log10(cond)) + 7)
    for _ in range(20):
        Q, _ = np.linalg.qr(rng.randn(6, 6))
        s = np.logspace(0, -math.log10(cond), 6) * 10.0 ** rng.uniform(-2, 4)
        A = (Q * s) @ Q.T
        A = 0.5 * (A + A.T)
        g = rng.randn(6) * 10.0 ** rng.uniform(-3, 1)
        xi, reason = TW.cholesky_solve(pack(A, g))
        assert reason is None
        ref = -np.linalg.solve(A, g)
        err = np.linalg.norm(np.array(xi) - ref) / np.linalg.norm(ref)
        assert err <= 50 * cond * EPS, (cond, err)


def test_a_zero_or_singular_system_is_lost():
    assert TW.cholesky_solve(np.zeros(27)) == (None, "pivot")
    # J never moves along the third coordinate (a fronto-parallel plane's rotation about the optical axis): the third
    # pivot is exactly 0
    rng = np.random.RandomState(3)
    J = rng.randn(500, 6)
    J[:, 2] = 0.0
    A = J.T @ J
    assert TW.cholesky_solve(pack(A, J.T @ rng.randn(500))) == (None, "pivot")
    # a negative pivot
    A = np.eye(6)
    A[4, 4] = -1e-12
    assert TW.cholesky_solve(pack(A, np.ones(6))) == (None, "pivot")


def test_loss_rule_is_the_fp32_fraction_widened_to_double():
    """inliers < double(float(min_inlier_fraction)) * valid: 0.1f is 0.10000000149..., so 10 of 100 is lost, and the
    comparison is strict, so 25 of 100 at 0.25 is not."""
    tp = TrackParams.defaults()
    A, g = np.eye(6), np.full(6, 1e-3)
    pose = np.eye(4, dtype=np.float32)[:3]
    tp.min_inlier_fraction = 0.1
    assert TW.solve_step(pack(A, g), 10, 100, pose, 2, tp)["reason"] == "inliers"
    assert not TW.solve_step(pack(A, g), 11, 100, pose, 2, tp)["lost"]
    tp.min_inlier_fraction = 0.25
    assert not TW.solve_step(pack(A, g), 25, 100, pose, 2, tp)["lost"]
    assert TW.solve_step(pack(A, g), 24, 100, pose, 2, tp)["reason"] == "inliers"
    # 0 of 0 valid pixels passes the rule; the zero system then loses by its pivot
    tp.min_inlier_fraction = 0.0
    assert TW.solve_step(np.zeros(27), 0, 0, pose, 0, tp)["reason"] == "pivot"


def test_convergence_rule_is_on_the_norms():
    """|omega| < convergence_rotation and |v| < convergence_translation, not their squares: a step of norm 3e-6 in
    both does not end a level at thresholds of 1e-5 squared, and does at 1e-5."""
    tp = TrackParams.defaults()
    pose = np.eye(4, dtype=np.float32)[:3]
    xi = np.array([2e-6, -2e-6, 1e-6, 1e-6, 2e-6, -2e-6])
    g = -xi   # A = I
    step = TW.solve_step(pack(np.eye(6), g), 100, 100, pose, 1, tp)
    assert step["converged"] and np.allclose(step["xi"], xi, rtol=1e-15, atol=0)
    tp.convergence_rotation = 2.9e-6
    assert not TW.solve_step(pack(np.eye(6), g), 100, 100, pose, 1, tp)["converged"]
    tp.convergence_rotation, tp.convergence_translation = 1e-5, 2.9e-6
    assert not TW.solve_step(pack(np.eye(6), g), 100, 100, pose, 1, tp)["converged"]


# ---- the SE(3) increment ---------------------------------------------------------------------------------------------
THETAS = [0.0, 1e-9, 9.999e-5, 1e-4, 1.0001e-4, 0.01, 0.5, 3.1]


def twist_exp(xi):
    X = np.zeros((4, 4))
    X[:3, :3] = TW.skew(xi[:3])
    X[:3, 3] = xi[3:]
    return expm(X)[:3]


def translation_bound(theta, v):
    """The increment's translation error: 1e-15 relative, plus the cancellation of its trig branch, where
    B = (1 - cos t) / t^2 carries cos's rounding divided by t^2 into V = I + B K + Cc K^2, i.e. ~eps |v| / t (7e-14
    relative at t = 1e-4; 1e-6 of an fp32 ulp, so the fp32 pose the kernel rounds to does not see it)."""
    extra = 2 * EPS / theta if theta >= 1e-4 else 0.0
    return (1e-15 + extra) * np.linalg.norm(v)


@pytest.mark.parametrize("theta", THETAS)
def test_increment_matches_expm(theta):
    rng = np.random.RandomState(int(theta * 1e4) % 1000 + 11)
    for _ in range(10):
        axis = rng.randn(3)
        axis /= np.linalg.norm(axis)
        xi = np.concatenate([theta * axis, rng.randn(3) * 0.05])
        got = np.array(TW.apply_increment(xi, np.eye(4)[:3])).reshape(3, 4)
        ref = twist_exp(xi)
        assert np.abs(got[:, :3] - ref[:, :3]).max() <= 1e-15, theta
        assert np.abs(got[:, 3] - ref[:, 3]).max() <= translation_bound(theta, xi[3:]), theta
        # applied to a pose: exp(xi) * pose
        P = offset(rng.randn(3) * 20, rng.randn(3))
        got = np.array(TW.apply_increment(xi, P)).reshape(3, 4)
        want = ref[:, :3] @ P
        want[:, 3] += ref[:, 3]
        assert np.abs(got - want).max() <= 4e-15 + translation_bound(theta, xi[3:])


def test_increment_branches_agree_at_the_switch():
    rng = np.random.RandomState(5)
    axis = rng.randn(3)
    axis /= np.linalg.norm(axis)
    v = rng.randn(3) * 0.05
    below = math.nextafter(1e-4, 0.0)
    a = np.array(TW.apply_increment(np.concatenate([below * axis, v]), np.eye(4)[:3])).reshape(3, 4)
    # the smallest rotation that takes the trig branch
    theta = 1e-4
    while math.sqrt(sum((theta * c) ** 2 for c in axis)) < 1e-4:
        theta = math.nextafter(theta, 1.0)
    b = np.array(TW.apply_increment(np.concatenate([theta * axis, v]), np.eye(4)[:3])).reshape(3, 4)
    assert np.abs(a[:, :3] - b[:, :3]).max() <= 1e-15
    assert np.abs(a[:, 3] - b[:, 3]).max() <= 2 * translation_bound(1e-4, v)


def test_se3_exp_rotation_is_rodrigues():
    rv = np.array([0.3, -0.2, 0.25])
    T = TW.se3_exp(np.concatenate([rv, [0.1, 0.2, 0.3]]))
    assert np.abs(T[:, :3] - Rotation.from_rotvec(rv).as_matrix()).max() <= 1e-15


# ---- the clear rule --------------------------------------------------------------------------------------------------
def test_clear_rule():
    """A generic step is clear; a step whose translation is put on an fp32 rounding midpoint, where an ulp of sin or
    cos decides the rounding, is not; the polynomial branch has no inexact input."""
    pose = np.eye(4, dtype=np.float32)[:3]
    xi = [0.004, -0.006, 0.007, 0.01, 0.5, -0.4]
    assert TW.step_is_clear(xi, pose)
    target = float(np.float32(0.01))
    target = 0.5 * (target + float(np.nextafter(np.float32(target), np.float32(1))))   # an fp32 midpoint
    for _ in range(6):   # t = V v with V_00 = 1 - O(theta^2): Newton steps on v_x with slope 1
        xi[3] += target - TW.apply_increment(xi, pose)[3]
    assert abs(TW.apply_increment(xi, pose)[3] - target) <= 4 * math.ulp(target)
    assert not TW.step_is_clear(xi, pose)
    step = TW.solve_step(pack(np.eye(6), -np.array(xi)), 100, 100, pose, 0, TrackParams.defaults())
    assert not step["clear"]
    assert TW.step_is_clear([1e-6, 2e-6, -3e-6, 0.01, 0.02, 0.03], pose)


# ---- the host pose code ----------------------------------------------------------------------------------------------
def polar(M):
    U, _, Vt = np.linalg.svd(M)
    return U @ Vt


def perturbed_guesses():
    rng = np.random.RandomState(9)
    out = []
    for _ in range(5):
        T = offset(rng.randn(3) * 40, rng.randn(3))
        out.append(("near", T.astype(np.float32).astype(np.float64)))
        S = T.copy()
        S[:, :3] *= 1.002
        S[0, 1] += 0.001
        out.append(("scaled_sheared", S))
        B = T.copy()
        B[:, :3] *= 1.5
        out.append(("scale_1.5", B))
    return out


@pytest.mark.parametrize("kind", ["near", "scaled_sheared", "scale_1.5"])
def test_project_to_rigid_is_the_polar_factor(kind):
    for name, T in perturbed_guesses():
        if name != kind:
            continue
        P = TW.project_to_rigid(T)
        assert np.abs(P[:, :3] - polar(T[:, :3])).max() <= 1e-14
        assert np.array_equal(P[:, 3], T[:, 3])


def test_project_to_rigid_fixed_points_and_refusals():
    for M in (np.eye(3), np.array([[0.0, -1, 0], [1, 0, 0], [0, 0, 1]]), np.array([[0.0, 0, 1], [1, 0, 0], [0, 1, 0]])):
        T = np.concatenate([M, [[0.5], [-1.0], [2.0]]], axis=1)
        assert np.array_equal(TW.project_to_rigid(T), T)
    R = Rotation.from_rotvec([0.3, -1.1, 0.7]).as_matrix()
    P = TW.project_to_rigid(np.concatenate([R, np.zeros((3, 1))], axis=1))
    assert np.abs(P[:, :3] - R).max() <= 4 * EPS
    mirrored = np.eye(4)[:3].copy()
    mirrored[0, 0] = -1.0
    assert TW.project_to_rigid(mirrored) is None
    assert TW.project_to_rigid(np.zeros((3, 4))) is None


def test_invert_and_compose_rigid():
    rng = np.random.RandomState(4)
    for _ in range(10):
        A = TW.project_to_rigid(offset(rng.randn(3) * 30, rng.randn(3) * 2))
        B = TW.project_to_rigid(offset(rng.randn(3) * 30, rng.randn(3) * 2))
        assert np.abs(TW.compose_rigid(A, B) - TW.compose(A, B)).max() <= 1e-14
        assert np.abs(TW.invert_rigid(A) - TW.invert(A)).max() <= 1e-14
        assert np.abs(TW.compose_rigid(TW.invert_rigid(A), A) - np.eye(4)[:3]).max() <= 1e-14


# ---- the whole walk on the plane scenes ------------------------------------------------------------------------------
def scene_walk(name, truth, tp):
    z, n = TW.render_planes(TW.SCENES[name], CAM, np.eye(4)[:3])
    model_depth = np.where(np.isfinite(z), z, 0).astype(np.float32)
    model_normal = n.astype(np.float32)
    live = [TW.quantize(TW.render_planes(TW.SCENES[name], TW.scaled(CAM, l), truth)[0]) for l in range(tp.levels)]

    def linearize_level(level, pose):
        lin = TW.linearize(live[level], 5000.0, TW.scaled(CAM, level)[2:], model_depth, model_normal, CAM[2:],
                           pose.reshape(3, 4))
        return dict(system=lin["system"], inliers=lin["inliers"], valid=lin["valid"], r2=lin["r2"])

    return TW.run_schedule(np.eye(4, dtype=np.float32)[:3], tp, linearize_level)


@pytest.mark.parametrize("scene", sorted(TW.SCENES))
def test_walk_on_the_plane_scenes(scene):
    truth = offset((1.0, -1.5, 0.8), (0.02, -0.015, 0.01)).astype(np.float32)
    tp = TrackParams.defaults()
    pose, lost, iterations, stats, trace = scene_walk(scene, truth, tp)
    applied = [s for s in trace if not s["skipped"]]
    assert all(s["clear"] for s in applied)
    assert len(trace) == sum(tp.iterations[:tp.levels])
    ends = [s["level"] for s in applied if s["converged"]]
    print(f"{scene}: lost {lost}, {iterations} steps, levels ended by convergence {ends}, "
          f"level-0 inliers {stats and stats['inliers']}")
    if scene == "corner":
        assert not lost and ends, "the corner converges"
        # a converged level's remaining steps are no-ops, and the next level starts afresh
        for level in ends:
            at = [s for s in trace if s["level"] == level]
            k = next(i for i, s in enumerate(at) if not s["skipped"] and s["converged"])
            assert all(s["skipped"] for s in at[k + 1:])
        dt, dr = TW.pose_error(pose.reshape(3, 4), truth)
        assert dt < 1e-3 and dr < 0.05, (dt, dr)
        assert iterations == len(applied)
    elif scene == "fronto_parallel":
        # one plane facing the camera: its normal has no x or y component, so rotation about the optical axis and
        # the two in-plane translations leave J^T J with an exactly zero pivot on the first step
        assert lost and applied[0]["reason"] == "pivot" and len(applied) == 1 and iterations == 0
        assert all(s["skipped"] for s in trace[1:]) and stats is None


def test_walk_schedules_with_empty_levels():
    """A level with zero iterations is passed over, a schedule without level-0 steps has no level-0 statistics, and
    one step per level applies exactly one step per level."""
    truth = offset((1.0, -1.5, 0.8), (0.02, -0.015, 0.01)).astype(np.float32)
    tp = TrackParams.defaults()
    tp.levels, tp.iterations = 4, (type(tp.iterations))(0, 3, 0, 2)
    _, lost, iterations, stats, trace = scene_walk("corner", truth, tp)
    assert not lost and stats is None and [s["level"] for s in trace] == [3, 3, 1, 1, 1]
    assert iterations == sum(not s["skipped"] for s in trace)
    tp.iterations = (type(tp.iterations))(1, 1, 1, 1)
    _, lost, iterations, stats, trace = scene_walk("corner", truth, tp)
    assert not lost and iterations == 4 and [s["level"] for s in trace] == [3, 2, 1, 0] and stats["inliers"] > 0
    res = TW.level_stats(stats, rgbd=False)
    assert res["rms_residual"] == np.float32(math.sqrt(stats["r2"] / stats["inliers"]))
