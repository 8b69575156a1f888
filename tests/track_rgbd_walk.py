"""numpy restatement of sm_track_linearize_rgbd's photometric rules (include/surfel_b200.h, rules P1-P6) on top of
tests/track_walk.py's rules L and M: every per-pixel step in float32, one rounded operation at a time, in the order the
header states; the sums in float64. Also textured analytic scenes (track_walk.SCENES with an intensity texture in plane
coordinates) and a wall stream: a camera sliding in front of one textured wall, the case point-to-plane ICP cannot
track."""
from __future__ import annotations

import math

import numpy as np

from tests import track_walk as TW

f32 = np.float32
f64 = np.float64


# ---- P1-P3: intensity and the pyramids ---------------------------------------------------------------------------
def intensity(rgb):
    """P1 of a u8 [..., 3] image: ((0.299 r + 0.587 g) + 0.114 b) in float32."""
    c = np.asarray(rgb).astype(f32)
    return (f32(0.299) * c[..., 0] + f32(0.587) * c[..., 1]) + f32(0.114) * c[..., 2]


def downscale(I, width, height):
    """P2: one level of size width x height from I [h', w']; the clamped 2x2 average, every sum rounded."""
    h, w = I.shape
    x, y = np.arange(width), np.arange(height)
    x0, y0 = 2 * x, 2 * y
    assert x0.max() <= w - 1 and y0.max() <= h - 1, "an index passes the edge"
    x1, y1 = np.minimum(2 * x + 1, w - 1), np.minimum(2 * y + 1, h - 1)
    with np.errstate(invalid="ignore"):
        return ((I[y0][:, x0] + I[y0][:, x1]) + (I[y1][:, x0] + I[y1][:, x1])) * f32(0.25)


def pyramid(I0, cam, levels):
    """Levels 0..levels-1 from level 0 at cam = (width, height, fx, fy, cx, cy), at the sizes of Camera.scaled."""
    out = [np.asarray(I0, f32)]
    for l in range(1, levels):
        w, h = TW.scaled(cam, l)[:2]
        out.append(downscale(out[-1], w, h))
    return out


def model_intensity(color, depth):
    """P3 level 0: P1 of the model colour where the model depth is finite and > 0, NaN elsewhere."""
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(depth) & (depth > 0)
    return np.where(ok, intensity(color), f32(np.nan)).astype(f32)


# ---- P4-P6 ---------------------------------------------------------------------------------------------------------
def linearize(live, depth_scaling, live_cam, model_depth, model_normal, model_cam, T, live_I, model_I,
              photometric_weight, max_intensity_residual, min_gradient, max_point_distance=0.05,
              max_normal_angle_deg=20.0):
    """Rules L, M and P at one level. live_cam = (fx, fy, cx, cy) of the level (also the level's model camera for
    P4), model_cam = (fx, fy, cx, cy) of the handle (M2); live_I / model_I the level's pyramid images. Returns a dict:
    system (float64 [27], depth and photometric terms), magnitude (sum of |term| per entry), inliers, valid, r2,
    rc2, photometric_inliers, the depth-only system, and per photometric inlier in float32 J_c [k, 6], r_c [k], the
    live point p, the pixel (x, y), the bilinear cell (i, j)."""
    with np.errstate(all="ignore"):
        fx, fy, cx, cy = (f32(v) for v in live_cam)
        mfx, mfy, mcx, mcy = (f32(v) for v in model_cam)
        H, W = model_depth.shape
        p, n, valid = TW.live_points_normals(live, depth_scaling, fx, fy, cx, cy)
        ys, xs = np.nonzero(valid)
        p, n = p[valid], n[valid]
        # M1-M4, as track_walk.linearize states them
        pm = TW.transform(T, p)
        nl = TW.transform(T, n, translate=False)
        u = mfx * (pm[:, 0] / pm[:, 2]) + mcx
        v = mfy * (pm[:, 1] / pm[:, 2]) + mcy
        ok = (pm[:, 2] > f32(0)) & (u >= f32(0)) & (u < f32(W)) & (v >= f32(0)) & (v < f32(H))
        ix = np.where(ok, u, 0).astype(np.int64)
        iy = np.where(ok, v, 0).astype(np.int64)
        dm = model_depth[iy, ix].astype(f32)
        ok &= np.isfinite(dm) & (dm > f32(0))
        nm, nok = TW.normalize(model_normal[iy, ix].astype(f32))
        ok &= nok
        q = np.stack([dm * TW.ray(ix, mcx, mfx), dm * TW.ray(iy, mcy, mfy), dm], axis=-1)
        nm = np.where((TW.dot(nm, q) > f32(0))[:, None], -nm, nm)
        e = pm - q
        d2 = f32(max_point_distance) * f32(max_point_distance)
        cos_angle = f32(math.cos(float(f32(max_normal_angle_deg)) * math.pi / 180.0))
        ok &= (TW.dot(e, e) <= d2) & (TW.dot(nl, nm) >= cos_angle)
        r = TW.dot(nm, e)[ok]
        J = np.concatenate([TW.cross(pm, nm), nm], axis=-1)[ok]
        pm, p, xs, ys = pm[ok], p[ok], xs[ok], ys[ok]
        # P4
        hl, wl = model_I.shape
        s = (fx * (pm[:, 0] / pm[:, 2]) + cx) - f32(0.5)
        t = (fy * (pm[:, 1] / pm[:, 2]) + cy) - f32(0.5)
        cok = (s >= f32(0)) & (s < f32(wl - 1)) & (t >= f32(0)) & (t < f32(hl - 1))
        i = np.where(cok, s, 0).astype(np.int64)
        j = np.where(cok, t, 0).astype(np.int64)
        a = s - i.astype(f32)
        b = t - j.astype(f32)
        I00, I10, I01, I11 = model_I[j, i], model_I[j, i + 1], model_I[j + 1, i], model_I[j + 1, i + 1]
        cok &= np.isfinite(I00) & np.isfinite(I10) & np.isfinite(I01) & np.isfinite(I11)
        oa, ob = f32(1) - a, f32(1) - b
        im = (oa * I00 + a * I10) * ob + (oa * I01 + a * I11) * b
        gx = ob * (I10 - I00) + b * (I11 - I01)
        gy = oa * (I01 - I00) + a * (I11 - I10)
        rc = im - live_I[ys, xs]
        g2 = f32(min_gradient) * f32(min_gradient)
        cok &= (np.abs(rc) <= f32(max_intensity_residual)) & (gx * gx + gy * gy >= g2)
        # P5
        ga, gb = gx * fx, gy * fy
        iz = f32(1) / pm[:, 2]
        w = np.stack([ga * iz, gb * iz, -(((ga * pm[:, 0] + gb * pm[:, 1]) * iz) * iz)], axis=-1)
        Jc = np.concatenate([TW.cross(pm, w), w], axis=-1)[cok]
        rc = rc[cok]
    # P6
    J64, r64 = J.astype(f64), r.astype(f64)
    Jc64, rc64 = Jc.astype(f64), rc.astype(f64)
    lam2 = f64(f32(photometric_weight)) * f64(f32(photometric_weight))
    depth_terms = [J64[:, k] * J64[:, m] for k in range(6) for m in range(k, 6)] + [J64[:, k] * r64 for k in range(6)]
    photo_terms = [lam2 * (Jc64[:, k] * Jc64[:, m]) for k in range(6) for m in range(k, 6)] + \
                  [lam2 * (Jc64[:, k] * rc64) for k in range(6)]
    depth_system = np.array([t_.sum() for t_ in depth_terms], f64)
    system = depth_system + np.array([t_.sum() for t_ in photo_terms], f64)
    magnitude = np.array([np.abs(d_).sum() + np.abs(p_).sum() for d_, p_ in zip(depth_terms, photo_terms)], f64)
    return dict(system=system, depth_system=depth_system, magnitude=magnitude, inliers=int(ok.sum()),
                valid=int(valid.sum()), r2=float((r64 * r64).sum()), rc2=float((rc64 * rc64).sum()),
                photometric_inliers=int(cok.sum()), Jc=Jc, rc=rc, p=p[cok], x=xs[cok], y=ys[cok], i=i[cok], j=j[cok])


def photometric_residual(p_live, T, model_I, level_cam, i, j, live_value):
    """r_c of P4 in float64 for one live point inside the fixed bilinear cell (i, j): the function whose derivative
    J_c of P5 describes."""
    fx, fy, cx, cy = (float(v) for v in level_cam)
    T = np.asarray(T, f64).reshape(3, 4)
    pm = T[:, :3] @ p_live + T[:, 3]
    a = fx * pm[0] / pm[2] + cx - 0.5 - i
    b = fy * pm[1] / pm[2] + cy - 0.5 - j
    I = model_I.astype(f64)
    im = ((1 - a) * I[j, i] + a * I[j, i + 1]) * (1 - b) + ((1 - a) * I[j + 1, i] + a * I[j + 1, i + 1]) * b
    return float(im - live_value)


def gauss_newton(live, depth_scaling, live_cam, model_depth, model_normal, model_cam, T0, live_I, model_I,
                 photometric_weight, max_intensity_residual=40.0, min_gradient=2.0, iterations=10):
    """Plain Gauss-Newton on the restatement at one level: T <- exp(xi) T, pose rounded to float32."""
    T = np.asarray(T0, f32).reshape(3, 4)
    for _ in range(iterations):
        lin = linearize(live, depth_scaling, live_cam, model_depth, model_normal, model_cam, T, live_I, model_I,
                        photometric_weight, max_intensity_residual, min_gradient)
        A, b = TW.unpack(lin["system"])
        T = TW.compose(TW.se3_exp(-np.linalg.solve(A, b)), T).astype(f32)
    return T


# ---- textured analytic scenes --------------------------------------------------------------------------------------
def tangent_basis(n):
    n = np.asarray(n, f64)
    helper = np.array([1.0, 0.0, 0.0]) if abs(n[0]) < 0.9 else np.array([0.0, 1.0, 0.0])
    u = np.cross(n, helper)
    u /= np.linalg.norm(u)
    return u, np.cross(n, u)


def texture(a, b):
    """u8 [..., 3] colour at plane coordinates (a, b) in metres: a smooth sine sum plus a coarse checker."""
    smooth = 40.0 * np.sin(9.0 * a + 4.0 * b) + 30.0 * np.sin(-7.0 * a + 13.0 * b) + 20.0 * np.sin(31.0 * a + 17.0 * b)
    checker = 15.0 * (1 - 2 * ((np.floor(a / 0.2) + np.floor(b / 0.2)) % 2))
    v = 125.0 + smooth + checker
    rgb = np.stack([v, 0.9 * v + 10.0, 0.8 * v + 20.0], axis=-1)
    return np.clip(np.round(rgb), 0, 255).astype(np.uint8)


def render_textured_planes(planes, cam, global_T_camera):
    """track_walk.render_planes plus the colour [H, W, 3] u8 of the nearest plane's texture (black where no hit)."""
    w, h, fx, fy, cx, cy = cam
    T = np.asarray(global_T_camera, f64).reshape(3, 4)
    R, o = T[:, :3], T[:, 3]
    z, normal = TW.render_planes(planes, cam, global_T_camera)
    xs = (np.arange(w) + 0.5 - cx) / fx
    ys = (np.arange(h) + 0.5 - cy) / fy
    d = np.stack(np.broadcast_arrays(xs[None, :], ys[:, None], np.ones((h, w))), axis=-1) @ R.T
    color = np.zeros((h, w, 3), np.uint8)
    best = np.full((h, w), np.inf)
    for n, off in planes:
        n = np.asarray(n, f64)
        with np.errstate(all="ignore"):
            t = (off - n @ o) / (d @ n)
        hit = np.isfinite(t) & (t > 1e-6) & (t < best)
        best = np.where(hit, t, best)
        X = o + np.where(hit, t, 0)[..., None] * d
        u, v = tangent_basis(n)
        color = np.where(hit[..., None], texture(X @ u, X @ v), color)
    return z, normal, color


# ---- the wall stream -----------------------------------------------------------------------------------------------
WALL = [((0.0, 0.0, 1.0), 1.2)]   # the plane z = 1.2 m; the camera starts at the origin looking along +z


def wall_trajectory(frame_count):
    """[F, 3, 4] float64 camera-to-world poses at 30 Hz: a slide parallel to the wall at 0.25 m/s with a sinusoidal
    speed change, so the constant-velocity guess is off by up to about a centimetre, and small rotations (a few
    degrees about the wall normal, about one across the view)."""
    from scipy.spatial.transform import Rotation
    poses = np.zeros((frame_count, 3, 4))
    for k in range(frame_count):
        t = k / 30.0
        x = 0.25 * t + 0.12 * math.sin(2 * math.pi * 1.2 * t)
        y = 0.06 * math.sin(2 * math.pi * 0.9 * t + 1.0)
        rot = np.radians([1.0 * math.sin(2 * math.pi * 0.5 * t), 0.8 * math.sin(2 * math.pi * 0.6 * t + 2.0),
                          3.0 * math.sin(2 * math.pi * 0.7 * t)])
        poses[k, :, :3] = Rotation.from_rotvec(rot).as_matrix()
        poses[k, :, 3] = (x, y, 0.02 * math.sin(2 * math.pi * 0.4 * t))
    return poses


def wall_stream(cam, frame_count, depth_scaling=5000.0, seed=20261017):
    """(depth [F, H, W] u16, colour [F, H, W, 3] u8, poses [F, 3, 4] float64) of the wall seen along
    wall_trajectory, cam = (width, height, fx, fy, cx, cy). Depth noise is the synthetic stream's Kinect-like
    sigma(z) = 0.0012 + 0.0019 (z - 0.4)^2."""
    rng = np.random.RandomState(seed)
    poses = wall_trajectory(frame_count)
    w, h = cam[:2]
    depth = np.zeros((frame_count, h, w), np.uint16)
    color = np.zeros((frame_count, h, w, 3), np.uint8)
    for k in range(frame_count):
        z, _, rgb = render_textured_planes(WALL, cam, poses[k])
        sigma = 0.0012 + 0.0019 * (np.minimum(z, 10.0) - 0.4) ** 2
        depth[k] = TW.quantize(z + sigma * rng.standard_normal(z.shape), depth_scaling)
        color[k] = rgb
    return depth, color, poses
