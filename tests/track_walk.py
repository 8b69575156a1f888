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
    """[3, 4] float64 exp of xi = (omega, v): Rodrigues rotation, translation V v with the SE(3) left Jacobian V."""
    w, v = np.asarray(xi[:3], f64), np.asarray(xi[3:], f64)
    theta2 = float(w @ w)
    theta = math.sqrt(theta2)
    if theta < 1e-4:
        A, B, Cc = 1.0 - theta2 / 6.0, 0.5 - theta2 / 24.0, 1.0 / 6.0 - theta2 / 120.0
    else:
        A, B, Cc = math.sin(theta) / theta, (1.0 - math.cos(theta)) / theta2, (theta - math.sin(theta)) / (theta2 * theta)
    K = skew(w)
    K2 = K @ K
    R = np.eye(3) + A * K + B * K2
    V = np.eye(3) + B * K + Cc * K2
    return np.concatenate([R, (V @ v)[:, None]], axis=1)


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


def nearest_rotation(T):
    """The 3x4 pose with its 3x3 part replaced by the nearest rotation: the Newton polar iteration
    R <- (R + R^-T) / 2 in float64 that sm_track_frame applies to the guess, the model pose and the result."""
    T = np.asarray(T, f64).reshape(3, 4).copy()
    R = T[:, :3]
    for _ in range(8):
        R = 0.5 * (R + np.linalg.inv(R).T)
    T[:, :3] = R
    return T


def live_view(depth, depth_scaling, cam):
    """Rule L's level-0 view of a u16 image: (z where the pixel is valid else 0, unit normals), float32."""
    p, n, valid = live_points_normals(depth, depth_scaling, *(f32(v) for v in cam[2:]))
    return np.where(valid, p[..., 2], f32(0)).astype(f32), n


def track_previous_frame_chain(depths, first_pose, cam, depth_scaling=5000.0, iterations=8, project=True):
    """sm_track_frame's pose bookkeeping for a pose-free sequence tracked frame to frame at level 0: each frame from
    the constant-velocity guess T_{k-1} T_{k-2}^-1 T_{k-1} against the previous frame's view at the pose returned
    for it. `project` applies the nearest-rotation projection of the library; without it the fp32 poses drift off
    SO(3). Returns the float32 [3, 4] poses."""
    fix = nearest_rotation if project else (lambda T: np.asarray(T, f64).reshape(3, 4))
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
