"""numpy restatement of sm_track_linearize's per-pixel rules (include/surfel_b200.h, rules L and M): every per-pixel
step in float32, one rounded operation at a time, in the order the header states; the sums in float64. Also the SE(3)
exponential of the solve, a plain Gauss-Newton loop on top of the restatement, and analytic plane scenes to run
both on."""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32
f64 = np.float64


def scaled(cam, level: int):
    """(width, height, fx, fy, cx, cy) of Camera.scaled(level) for cam = (width, height, fx, fy, cx, cy)."""
    w, h, fx, fy, cx, cy = cam
    factor = f32(1.0) / f32(2.0 ** level)
    return (int(float(factor) * w + 0.5), int(float(factor) * h + 0.5), f32(fx) * factor, f32(fy) * factor,
            f32(cx) * factor, f32(cy) * factor)


def ray(p, c, f):
    return ((np.asarray(p).astype(f32) + f32(0.5)) - f32(c)) / f32(f)


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def normalize(n):
    """(n * (1 / sqrt(n.n)), ok) with ok = n.n finite and > 0."""
    len2 = dot(n, n)
    ok = np.isfinite(len2) & (len2 > f32(0))
    inv = f32(1) / np.sqrt(np.where(ok, len2, f32(1)))
    return n * inv[..., None], ok


def live_points_normals(live, depth_scaling, fx, fy, cx, cy):
    """Rules L1-L2 on an [h, w] u16 image: (p [h, w, 3], n [h, w, 3], valid [h, w]) in float32."""
    h, w = live.shape
    z = live.astype(f32) * (f32(1) / f32(depth_scaling))
    P = np.stack([z * ray(np.arange(w), cx, fx)[None, :], z * ray(np.arange(h), cy, fy)[:, None], z], axis=-1)
    valid = np.zeros((h, w), bool)
    n = np.zeros((h, w, 3), f32)
    nz = live != 0
    valid[1:-1, 1:-1] = nz[1:-1, 1:-1] & nz[1:-1, :-2] & nz[1:-1, 2:] & nz[:-2, 1:-1] & nz[2:, 1:-1]
    a = P[1:-1, 2:] - P[1:-1, :-2]
    b = P[2:, 1:-1] - P[:-2, 1:-1]
    ni, ok = normalize(cross(b, a))
    valid[1:-1, 1:-1] &= ok
    n[1:-1, 1:-1] = ni
    return P, n, valid


def transform(T, p, translate=True):
    T = np.asarray(T, f32).reshape(3, 4)
    rows = [(T[i, 0] * p[..., 0] + T[i, 1] * p[..., 1]) + T[i, 2] * p[..., 2] for i in range(3)]
    if translate:
        rows = [rows[i] + T[i, 3] for i in range(3)]
    return np.stack(rows, axis=-1)


def linearize(live, depth_scaling, live_cam, model_depth, model_normal, model_cam, T, max_point_distance=0.05,
              max_normal_angle_deg=20.0):
    """Rules L and M. live_cam / model_cam = (fx, fy, cx, cy). Returns a dict: system (float64 [27]), magnitude
    (sum of |term| per entry: the scale of fp64 summation error), inliers, valid, r2 and, per inlier in float32,
    J [k, 6], r [k], the live point p, the model point q and the camera-facing model normal n."""
    with np.errstate(all="ignore"):
        fx, fy, cx, cy = (f32(v) for v in live_cam)
        mfx, mfy, mcx, mcy = (f32(v) for v in model_cam)
        H, W = model_depth.shape
        p, n, valid = live_points_normals(live, depth_scaling, fx, fy, cx, cy)
        p, n = p[valid], n[valid]
        pm = transform(T, p)
        nl = transform(T, n, translate=False)
        u = mfx * (pm[:, 0] / pm[:, 2]) + mcx
        v = mfy * (pm[:, 1] / pm[:, 2]) + mcy
        ok = (pm[:, 2] > f32(0)) & (u >= f32(0)) & (u < f32(W)) & (v >= f32(0)) & (v < f32(H))
        ix = np.where(ok, u, 0).astype(np.int64)
        iy = np.where(ok, v, 0).astype(np.int64)
        dm = model_depth[iy, ix].astype(f32)
        ok &= np.isfinite(dm) & (dm > f32(0))
        nm, nok = normalize(model_normal[iy, ix].astype(f32))
        ok &= nok
        q = np.stack([dm * ray(ix, mcx, mfx), dm * ray(iy, mcy, mfy), dm], axis=-1)
        nm = np.where((dot(nm, q) > f32(0))[:, None], -nm, nm)
        e = pm - q
        d2 = f32(max_point_distance) * f32(max_point_distance)
        cos_angle = f32(math.cos(float(f32(max_normal_angle_deg)) * math.pi / 180.0))
        ok &= (dot(e, e) <= d2) & (dot(nl, nm) >= cos_angle)
        r = dot(nm, e)[ok]
        J = np.concatenate([cross(pm, nm), nm], axis=-1)[ok]
        p, q, nm = p[ok], q[ok], nm[ok]
    J64, r64 = J.astype(f64), r.astype(f64)
    terms = [J64[:, i] * J64[:, j] for i in range(6) for j in range(i, 6)] + [J64[:, i] * r64 for i in range(6)]
    system = np.array([t.sum() for t in terms], f64)
    magnitude = np.array([np.abs(t).sum() for t in terms], f64)
    return dict(system=system, magnitude=magnitude, inliers=int(ok.sum()), valid=int(valid.sum()),
                r2=float((r64 * r64).sum()), J=J, r=r, p=p, q=q, n=nm)


def unpack(system):
    """(J^T J [6, 6], J^T r [6]) from the 27 sums."""
    A = np.zeros((6, 6))
    k = 0
    for i in range(6):
        for j in range(i, 6):
            A[i, j] = A[j, i] = system[k]
            k += 1
    return A, np.asarray(system[21:27], f64)


def skew(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def se3_exp(xi):
    """[3, 4] float64 exp of xi = (omega, v): Rodrigues rotation, translation V v with the SE(3) left Jacobian V, in
    apply_increment's order (increment below)."""
    R, t = increment(xi)
    return np.concatenate([np.array(R), np.array(t)[:, None]], axis=1)


def compose(a, b):
    a, b = np.asarray(a, f64).reshape(3, 4), np.asarray(b, f64).reshape(3, 4)
    return np.concatenate([a[:, :3] @ b[:, :3], (a[:, :3] @ b[:, 3] + a[:, 3])[:, None]], axis=1)


def invert(T):
    T = np.asarray(T, f64).reshape(3, 4)
    R = T[:, :3].T
    return np.concatenate([R, (-R @ T[:, 3])[:, None]], axis=1)


def pose_error(a, b):
    """(translation error in metres, rotation error in degrees) between two 3x4 poses; the angle from atan2 of its
    sine and cosine (acos of the trace alone has a floor of ~0.02 degrees for fp32 matrices)."""
    a, b = np.asarray(a, f64).reshape(3, 4), np.asarray(b, f64).reshape(3, 4)
    R = a[:, :3] @ b[:, :3].T
    s = 0.5 * np.linalg.norm([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return float(np.linalg.norm(a[:, 3] - b[:, 3])), math.degrees(math.atan2(s, (np.trace(R) - 1) / 2))


def gauss_newton(live, depth_scaling, live_cam, model_depth, model_normal, model_cam, T0, iterations=10, **gates):
    """Plain Gauss-Newton on the restatement: T <- exp(xi) T, xi = -(J^T J)^-1 J^T r, pose rounded to float32."""
    T = np.asarray(T0, f32).reshape(3, 4)
    for _ in range(iterations):
        lin = linearize(live, depth_scaling, live_cam, model_depth, model_normal, model_cam, T, **gates)
        A, b = unpack(lin["system"])
        xi = -np.linalg.solve(A, b)
        T = compose(se3_exp(xi), T).astype(f32)
    return T


def residual(p_live, T, n_model, q):
    """r = n.(T p - q) in float64 for one live point: the function whose Jacobian J = [T p x n, n] describes."""
    T = np.asarray(T, f64).reshape(3, 4)
    return float(n_model @ (T[:, :3] @ p_live + T[:, 3] - q))


# ---- analytic plane scenes ---------------------------------------------------------------------------------------
# A plane is (unit normal n, offset d) with n.X = d in world coordinates.
SCENES = {
    "fronto_parallel": [((0.0, 0.0, 1.0), 2.0)],
    "tilted": [(tuple(np.array([0.3, -0.2, 1.0]) / np.linalg.norm([0.3, -0.2, 1.0])), 1.8)],
    # the inside of a three-plane corner, each plane 30-35 degrees off the optical axis
    "corner": [(tuple(np.array(n) / np.linalg.norm(n)), d)
               for n, d in (((0.6, 0.0, 1.0), 1.6), ((-0.6, 0.0, 1.0), 1.6), ((0.0, -0.7, 1.0), 1.5))],
}


def render_planes(planes, cam, global_T_camera):
    """z-depth [H, W] float64 (inf = no hit) and the camera-frame normal [H, W, 3] of the nearest plane, through the
    pixel-centre rays of cam = (width, height, fx, fy, cx, cy)."""
    w, h, fx, fy, cx, cy = cam
    T = np.asarray(global_T_camera, f64).reshape(3, 4)
    R, o = T[:, :3], T[:, 3]
    xs = (np.arange(w) + 0.5 - cx) / fx
    ys = (np.arange(h) + 0.5 - cy) / fy
    d_cam = np.stack(np.broadcast_arrays(xs[None, :], ys[:, None], np.ones((h, w))), axis=-1)
    d = d_cam @ R.T
    best = np.full((h, w), np.inf)
    normal = np.zeros((h, w, 3))
    for n, off in planes:
        n = np.asarray(n, f64)
        den = d @ n
        with np.errstate(all="ignore"):
            t = (off - n @ o) / den
        hit = np.isfinite(t) & (t > 1e-6) & (t < best)
        best = np.where(hit, t, best)
        normal = np.where(hit[..., None], (R.T @ n)[None, None, :], normal)
    return best, normal


def quantize(z, depth_scaling=5000.0):
    ok = np.isfinite(z) & (z > 0) & (z * depth_scaling < 65535)
    return np.where(ok, np.round(np.where(ok, z, 0) * depth_scaling), 0).astype(np.uint16)


def live_view(depth, depth_scaling, cam):
    """Rule L's level-0 view of a u16 image: (z where the pixel is valid else 0, unit normals), float32."""
    p, n, valid = live_points_normals(depth, depth_scaling, *(f32(v) for v in cam[2:]))
    return np.where(valid, p[..., 2], f32(0)).astype(f32), n


def track_previous_frame_chain(depths, first_pose, cam, depth_scaling=5000.0, iterations=8, project=True):
    """sm_track_frame's pose bookkeeping for a pose-free sequence tracked frame to frame at level 0: each frame from
    the constant-velocity guess T_{k-1} T_{k-2}^-1 T_{k-1} against the previous frame's view at the pose returned
    for it. `project` applies the nearest-rotation projection of the library; without it the fp32 poses drift off
    SO(3). Returns the float32 [3, 4] poses."""
    fix = project_to_rigid if project else (lambda T: np.asarray(T, f64).reshape(3, 4))
    traj = [np.asarray(first_pose, f32).reshape(3, 4)]
    for k in range(1, len(depths)):
        if k < 2:
            guess = traj[-1]
        else:
            guess = compose(compose(traj[-1], invert(traj[-2])), traj[-1]).astype(f32)
        model_pose = fix(traj[-1])
        T = compose(invert(model_pose), fix(guess)).astype(f32)
        md, mn = live_view(depths[k - 1], depth_scaling, cam)
        for _ in range(iterations):
            lin = linearize(depths[k], depth_scaling, cam[2:], md, mn, cam[2:], T)
            A, b = unpack(lin["system"])
            T = compose(se3_exp(-np.linalg.solve(A, b)), T).astype(f32)
        traj.append(fix(compose(model_pose, T)).astype(f32))
    return traj


# ---- the frame: sm_track_frame's host pose code, solve and schedule, exactly -----------------------------------------
# track.cu is built with -fmad=false (device) and -ffp-contract=off (host), so every fp64 product and sum of the solve,
# apply_increment and the pose code is rounded on its own; Python floats repeat them bit for bit in the same order.
# The only inexact inputs are the device's double sin and cos (a few ulp; the clear rule of solve_step covers them).
def _flat12(T):
    return [float(v) for v in np.asarray(T, f64).reshape(-1)[:12]]


def project_to_rigid(T):
    """ProjectToRigid: the 3x3 part of a 3x4 pose replaced by its nearest rotation, 8 Newton steps
    R <- R / 2 + C / (2 det) with the cofactor matrix C (= det R^-T), in Python floats in track.cu's order. Returns the
    float64 [3, 4] pose, or None for a non-finite or non-positive determinant."""
    t = _flat12(T)
    for _ in range(8):
        a, b, c, d, e, f, g, h, i = t[0], t[1], t[2], t[4], t[5], t[6], t[8], t[9], t[10]
        C00, C01, C02 = e * i - f * h, f * g - d * i, d * h - e * g
        C10, C11, C12 = c * h - b * i, a * i - c * g, b * g - a * h
        C20, C21, C22 = b * f - c * e, c * d - a * f, a * e - b * d
        det = a * C00 + b * C01 + c * C02
        if not (det > 0.0) or not math.isfinite(det):
            return None
        s = 0.5 / det
        t[0], t[1], t[2] = 0.5 * a + s * C00, 0.5 * b + s * C01, 0.5 * c + s * C02
        t[4], t[5], t[6] = 0.5 * d + s * C10, 0.5 * e + s * C11, 0.5 * f + s * C12
        t[8], t[9], t[10] = 0.5 * g + s * C20, 0.5 * h + s * C21, 0.5 * i + s * C22
    return np.array(t, f64).reshape(3, 4)


def invert_rigid(T):
    """InvertRigid: [R^T | -(R^T t)] with each entry of R^T t summed over the rows in order."""
    m = _flat12(T)
    out = [0.0] * 12
    for i in range(3):
        for j in range(3):
            out[4 * i + j] = m[4 * j + i]
        out[4 * i + 3] = -(m[i] * m[3] + m[4 + i] * m[7] + m[8 + i] * m[11])
    return np.array(out, f64).reshape(3, 4)


def compose_rigid(A, B):
    """ComposeRigid: A * B of two 3x4 poses, ((a0 b0j + a1 b1j) + a2 b2j) (+ a3 for the translation)."""
    a, b = _flat12(A), _flat12(B)
    out = [0.0] * 12
    for i in range(3):
        for j in range(4):
            v = a[4 * i] * b[j] + a[4 * i + 1] * b[4 + j] + a[4 * i + 2] * b[8 + j]
            if j == 3:
                v += a[4 * i + 3]
            out[4 * i + j] = v
    return np.array(out, f64).reshape(3, 4)


def cholesky_solve(system):
    """The solve of k_track_solve on the 27 sums: Cholesky of J^T J in the kernel's loop order, then forward and back
    substitution for J^T J xi = -J^T r. Returns (xi as 6 floats, None), or (None, "pivot") for a pivot that is not
    > 0."""
    s = [float(v) for v in system]
    H = [[0.0] * 6 for _ in range(6)]
    g = [0.0] * 6
    k = 0
    for i in range(6):
        for j in range(i, 6):
            H[i][j] = H[j][i] = s[k]
            k += 1
        g[i] = s[21 + i]
    L = [[0.0] * 6 for _ in range(6)]
    for j in range(6):
        d = H[j][j]
        for m in range(j):
            d -= L[j][m] * L[j][m]
        if not (d > 0.0):
            return None, "pivot"
        L[j][j] = math.sqrt(d)
        for i in range(j + 1, 6):
            v = H[i][j]
            for m in range(j):
                v -= L[i][m] * L[j][m]
            L[i][j] = v / L[j][j]
    y = [0.0] * 6
    for i in range(6):
        v = -g[i]
        for m in range(i):
            v -= L[i][m] * y[m]
        y[i] = v / L[i][i]
    xi = [0.0] * 6
    for i in range(5, -1, -1):
        v = y[i]
        for m in range(i + 1, 6):
            v -= L[m][i] * xi[m]
        xi[i] = v / L[i][i]
    return xi, None


def increment(xi, sn=None, cs=None):
    """apply_increment's exp(xi): (R, t) as nested float lists, R = I + A K + B K^2 and t = V v with
    V = I + B K + Cc K^2, in the kernel's order. theta < 1e-4 takes the polynomial branch; otherwise sin and cos of
    theta are math.sin / math.cos unless given (the clear rule passes perturbed values)."""
    wx, wy, wz = float(xi[0]), float(xi[1]), float(xi[2])
    theta2 = wx * wx + wy * wy + wz * wz
    theta = math.sqrt(theta2)
    if theta < 1e-4:
        A = 1.0 - theta2 / 6.0
        B = 0.5 - theta2 / 24.0
        Cc = 1.0 / 6.0 - theta2 / 120.0
    else:
        sn = math.sin(theta) if sn is None else sn
        cs = math.cos(theta) if cs is None else cs
        A = sn / theta
        B = (1.0 - cs) / theta2
        Cc = (theta - sn) / (theta2 * theta)
    K = ((0.0, -wz, wy), (wz, 0.0, -wx), (-wy, wx, 0.0))
    K2 = [[K[i][0] * K[0][j] + K[i][1] * K[1][j] + K[i][2] * K[2][j] for j in range(3)] for i in range(3)]
    R = [[(float(i == j) + A * K[i][j]) + B * K2[i][j] for j in range(3)] for i in range(3)]
    V = [[(float(i == j) + B * K[i][j]) + Cc * K2[i][j] for j in range(3)] for i in range(3)]
    v = [float(x) for x in xi[3:6]]
    t = [V[i][0] * v[0] + V[i][1] * v[1] + V[i][2] * v[2] for i in range(3)]
    return R, t


def apply_increment(xi, pose, sn=None, cs=None):
    """exp(xi) * pose in fp64 before the rounding to fp32: 12 floats, ((R_i0 P_0j + R_i1 P_1j) + R_i2 P_2j) (+ t_i)."""
    R, t = increment(xi, sn, cs)
    P = _flat12(pose)
    out = [0.0] * 12
    for i in range(3):
        for j in range(4):
            v = R[i][0] * P[j] + R[i][1] * P[4 + j] + R[i][2] * P[8 + j]
            if j == 3:
                v += t[i]
            out[4 * i + j] = v
    return out


CLEAR_ULPS = 4   # the device's double sin / cos against the host's: a few ulp at most (CUDA: 2 ulp)


def _ulps(x, k):
    return math.nextafter(x, math.copysign(math.inf, k), steps=abs(k)) if k else x


def step_is_clear(xi, pose):
    """The clear rule: for theta >= 1e-4, the fp32 pose of exp(xi) * pose with sin and cos each moved by
    -CLEAR_ULPS..+CLEAR_ULPS ulp (A, B and Cc recomputed from them in the kernel's order: B and Cc are cancelling
    differences, so perturbing them directly would understate the spread) rounds to the same 12 fp32 values as with
    the host's own sin and cos. The polynomial branch has no inexact input and is always clear."""
    w = [float(v) for v in xi[:3]]
    theta = math.sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2])
    if theta < 1e-4:
        return True
    sn, cs = math.sin(theta), math.cos(theta)
    ref = np.array(apply_increment(xi, pose, sn, cs), f64).astype(f32)
    for ds in range(-CLEAR_ULPS, CLEAR_ULPS + 1):
        for dc in range(-CLEAR_ULPS, CLEAR_ULPS + 1):
            got = np.array(apply_increment(xi, pose, _ulps(sn, ds), _ulps(cs, dc)), f64).astype(f32)
            if not np.array_equal(got.view(np.uint32), ref.view(np.uint32)):
                return False
    return True


def solve_step(system, inliers, valid, pose, level, params):
    """solve<kT> of track.cu after the sum of the partial rows, for the 27 sums `system`, the inlier and valid
    counts, the fp32 pose `pose` (12 values) and params with min_inlier_fraction, convergence_rotation and
    convergence_translation (fp32 values, as in sm_track_params). Returns a dict: level, lost (bool), reason
    ("inliers", "pivot", "not finite" or None), xi (6 floats or None), pose (float32 [12]: the new pose, or the old
    one for a lost step), converged (the level ends) and clear (see step_is_clear)."""
    pose = np.asarray(pose, f32).reshape(-1)[:12].copy()
    out = dict(level=level, lost=True, reason=None, xi=None, pose=pose, converged=False, clear=True)
    if float(inliers) < float(f32(params.min_inlier_fraction)) * float(valid):
        out["reason"] = "inliers"
        return out
    xi, reason = cholesky_solve(system)
    if xi is None:
        out["reason"] = reason
        return out
    if not all(math.isfinite(v) for v in xi):
        out["reason"] = "not finite"
        return out
    w2 = xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2]
    v2 = xi[3] * xi[3] + xi[4] * xi[4] + xi[5] * xi[5]
    out.update(lost=False, xi=xi, pose=np.array(apply_increment(xi, pose), f64).astype(f32),
               converged=math.sqrt(w2) < float(f32(params.convergence_rotation)) and
               math.sqrt(v2) < float(f32(params.convergence_translation)),
               clear=step_is_clear(xi, pose))
    return out


def run_schedule(init_pose, params, linearize_level):
    """Step 4 of sm_track_frame: levels params.levels-1 down to 0, params.iterations[level] steps each, a converged
    level and every step after a loss a no-op. linearize_level(level, pose) returns the linearisation at the fp32
    pose: a dict with system (27 sums), inliers, valid, r2 and, for RGB-D, rc2 and photometric_inliers. Returns
    (pose float32 [12], lost, iterations, level-0 statistics of the last level-0 linearisation (or None), trace:
    one dict per scheduled step with the linearisation, solve_step's decisions and skipped = no-op)."""
    pose = np.asarray(init_pose, f32).reshape(-1)[:12].copy()
    lost, done_level, iterations, stats, trace = False, -1, 0, None, []
    for level in range(params.levels - 1, -1, -1):
        for _ in range(params.iterations[level]):
            if lost or done_level == level:
                trace.append(dict(level=level, skipped=True))
                continue
            lin = linearize_level(level, pose)
            if level == 0:
                stats = lin
            step = solve_step(lin["system"], lin["inliers"], lin["valid"], pose, level, params)
            step.update(skipped=False, linearization=lin)
            trace.append(step)
            if step["lost"]:
                lost = True
                continue
            pose = step["pose"]
            iterations += 1
            if step["converged"]:
                done_level = level
    return pose, lost, iterations, stats, trace


def level_stats(stats, rgbd):
    """inliers, valid_pixels, rms_residual (and photometric_inliers, rms_intensity) of sm_track_frame's result from the
    last level-0 linearisation (all 0 without one): rms = fp32(sqrt(sum / count)) for a count > 0."""
    out = dict(inliers=0, valid_pixels=0, rms_residual=f32(0))
    if rgbd:
        out.update(photometric_inliers=0, rms_intensity=f32(0))
    if stats is None:
        return out
    out.update(inliers=stats["inliers"], valid_pixels=stats["valid"],
               rms_residual=f32(math.sqrt(stats["r2"] / stats["inliers"])) if stats["inliers"] > 0 else f32(0))
    if rgbd:
        photo = stats.get("photometric_inliers", 0)
        out.update(photometric_inliers=photo,
                   rms_intensity=f32(math.sqrt(stats["rc2"] / photo)) if photo > 0 else f32(0))
    return out


def _assert_system_parity(gpu_system, gpu_inliers, ref, what):
    bound = 1e-9 * ref["magnitude"] + 1e-300
    bad = np.abs(np.asarray(gpu_system, f64) - ref["system"]) > bound
    assert gpu_inliers == ref["inliers"], (what, gpu_inliers, ref["inliers"])
    assert not bad.any(), (what, np.flatnonzero(bad), gpu_system[bad], ref["system"][bad])


def track_frame(rec, depth, guess, tp, pp, source="cloud", previous=None, color=None, rp=None):
    """Steps 1-5 of sm_track_frame (sm_track_frame_rgbd with `color`, a [H, W, 3] u8 CUDA tensor, and rp) on the
    handle `rec` (reconstruction.CUDASurfelReconstruction), for the raw depth (u16 CUDA tensor) and the 3x4 guess:
      1. the live pyramid from the product's bilateral filter (value_to_ignore 0, cutoff u16(depth_scaling *
         max_depth)) and median downscale of level 0 to the sizes of Camera.scaled;
      2. the model view: source "cloud" renders the cloud from fp32(inverse(project(guess))), near 0.1, far 100 (with
         colour for RGB-D); source "previous" uses `previous` (the "kept" entry this function returned for the
         handle's previous call): its rule-L view of the filtered level 0, its returned pose and its raw colour, which
         the model depth masks (P3);
      3. every step's system from the GPU (rec.track_linearize / track_linearize_rgbd), each checked against this
         restatement's linearize at 1e-9 x magnitude with the exact inlier count, then solve_step;
      4. the result: the guess unchanged if lost, else fp32(project(compose(model pose, pose))).
    The valid count and sum r^2 of a step are the restatement's (sm_track_linearize returns neither); rms_residual
    therefore comes from another summation order than the device's. Returns a dict: pose (float32 [3, 4]), tracked,
    iterations, the level-0 statistics (level_stats), trace (run_schedule's), clear (every applied step clear), and
    kept (the "previous" of the next call)."""
    import torch
    from surfelmeshing_b200 import reconstruction as Rn
    from tests import track_rgbd_walk as RW
    W, H = rec.width, rec.height
    cam = (W, H, f32(rec.fx), f32(rec.fy), f32(rec.cx), f32(rec.cy))
    rgbd = color is not None
    photometric = rgbd and float(rp.photometric_weight) > 0.0
    scale = float(pp.depth_scaling)
    if source == "previous":
        if previous is None:
            raise ValueError("source 'previous' needs an earlier call")
        if rgbd and not previous["rgbd"]:
            raise ValueError("source 'previous' with colour needs an earlier RGB-D call")
    guess32 = np.asarray(guess, f32).reshape(3, 4)
    # poses
    guess_d = project_to_rigid(guess32)
    if guess_d is None:
        raise ValueError("the rotation of the guess must have a positive determinant")
    global_T_model = guess_d if source == "cloud" else project_to_rigid(previous["pose"])
    if global_T_model is None:
        raise ValueError("the pose of the previous frame is not a rigid transform")
    model_T_global = invert_rigid(global_T_model)
    init = compose_rigid(model_T_global, guess_d).astype(f32)
    view_f = model_T_global.astype(f32)
    # 1. live pyramid
    level0 = torch.zeros_like(depth)
    Rn.BilateralFilteringAndDepthCutoffCUDA(None, pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor,
                                            0, pp.bilateral_filter_radius_factor,
                                            int(f32(pp.depth_scaling) * f32(pp.max_depth)), pp.depth_valid_region_radius,
                                            depth, level0)
    live_t = [level0] + [Rn.DownscaleUsingMedianWhileExcluding(None, 0, scaled(cam, l)[0], scaled(cam, l)[1], level0)
                         for l in range(1, tp.levels)]
    torch.cuda.synchronize()
    live = [t.cpu().numpy() for t in live_t]
    # 2. model view
    if source == "cloud":
        outs = ("depth", "normal", "color") if rgbd else ("depth", "normal")
        view = rec.render(view_f, W, H, cam[2], cam[3], cam[4], cam[5], near=0.1, far=100.0, outputs=outs)
        torch.cuda.synchronize()
        model_depth, model_normal = view["depth"].cpu().numpy(), view["normal"].cpu().numpy()
        model_color = view["color"].cpu().numpy() if rgbd else None
    else:
        model_depth, model_normal, model_color = previous["depth"], previous["normal"], previous["color"]
    md_t = torch.from_numpy(np.ascontiguousarray(model_depth)).cuda()
    mn_t = torch.from_numpy(np.ascontiguousarray(model_normal)).cuda()
    # 3. this frame's kept view
    kept_depth, kept_normal = live_view(live[0], scale, cam)
    live_color = color.cpu().numpy() if rgbd else None
    if photometric:
        mc_t = torch.from_numpy(np.ascontiguousarray(model_color)).cuda()
        live_I = RW.pyramid(RW.intensity(live_color), cam, tp.levels)
        model_I = RW.pyramid(RW.model_intensity(model_color, model_depth), cam, tp.levels)

    gates = dict(max_point_distance=float(tp.max_point_distance), max_normal_angle_deg=float(tp.max_normal_angle_deg))

    def linearize_level(level, pose):
        T = pose.reshape(3, 4)
        lc = scaled(cam, level)
        if photometric:
            system, rc2, inliers, photo = rec.track_linearize_rgbd(level, live_t[level], color, md_t, mn_t, mc_t, T,
                                                                   params=tp, rgbd=rp, depth_scaling=scale)
            ref = RW.linearize(live[level], scale, lc[2:], model_depth, model_normal, cam[2:], T, live_I[level],
                               model_I[level], rp.photometric_weight, rp.max_intensity_residual, rp.min_gradient,
                               **gates)
            _assert_system_parity(system, inliers, ref, ("rgbd", level))
            rc_terms = ref["rc"].astype(f64) ** 2
            assert photo == ref["photometric_inliers"], (level, photo, ref["photometric_inliers"])
            assert abs(rc2 - ref["rc2"]) <= 1e-9 * rc_terms.sum() + 1e-300, (level, rc2, ref["rc2"])
            return dict(system=system, inliers=inliers, valid=ref["valid"], r2=ref["r2"], rc2=rc2,
                        photometric_inliers=photo)
        system, inliers = rec.track_linearize(level, live_t[level], md_t, mn_t, T, params=tp, depth_scaling=scale)
        ref = linearize(live[level], scale, lc[2:], model_depth, model_normal, cam[2:], T, **gates)
        _assert_system_parity(system, inliers, ref, ("depth", level))
        return dict(system=system, inliers=inliers, valid=ref["valid"], r2=ref["r2"])

    pose, lost, iterations, stats, trace = run_schedule(init, tp, linearize_level)
    if lost:
        out = guess32.copy()
    else:
        out = project_to_rigid(compose_rigid(global_T_model, pose))
        assert out is not None
        out = out.astype(f32)
    result = dict(pose=out, tracked=0 if lost else 1, iterations=iterations, trace=trace,
                  clear=all(s["clear"] for s in trace if not s["skipped"]),
                  kept=dict(depth=kept_depth, normal=kept_normal, pose=out, rgbd=rgbd, color=live_color))
    result.update(level_stats(stats, rgbd))
    return result
