"""Float64 restatement of the bilateral filter with depth cutoff, the outlier fusion and the erosion of depth
pre-processing, from the u16 inputs and the fp32 parameters the library receives (eps = 2^-23).

Bilateral filter (cuda_depth_processing.cu:50-118 of the reference). A pixel outside the valid region
(float(u32 centre distance^2) > fp32 r^2), a centre equal to value_to_ignore and a centre above max_depth give
value_to_ignore; these are integer decisions and exact. Otherwise the value is v = sum w_i s_i / sum w_i over the
taps s_i != value_to_ignore of the disc dx^2 + dy^2 <= R^2 inside the image, R = int(fp32(radius_factor sigma_xy)
+ 0.5), with w_i = exp(u_i), u_i = -(dx^2 + dy^2) / (2 sigma_xy^2) - (c - s_i)^2 / (2 (c sigma_v)^2), and the output
is floor(v + 0.5).

How far the kernel's value can be from v, by its fp32 operation count:
- Weights. The exponent's two terms are both <= 0. The spatial one carries 2 sigma^2 (one rounding) and its
  approximate reciprocal (1 ulp): 1.5 eps. The range term carries -d^2 (eps/2), c sigma_v (eps/2), 2 av^2 (eps/2 more,
  so 1.5 eps), the approximate reciprocal (eps) and the product (eps/2): 3.5 eps. The fma that adds them rounds once
  (eps/2), the product with the fp32 log2(e) once more (eps/2, and the constant is 0.11 eps off): the argument of
  ex2 is within 4.7 eps |u_i| log2(e) of exact, so the weight is within 5 eps |u_i| of w_i relatively, before the
  approximate ex2 adds its own 2^-22 (budgeted as 4 eps). |u_i| reaches ~34 before w_i < 1e-15 stops mattering, so
  the argument costs up to ~160 eps of relative weight there. Below 2^-126 ex2 flushes to zero: such a weight is
  off by all of itself. Perturbing each weight by eta_i moves v by at most P = sum w_i eta_i |s_i - v| / sum w_i.
- Sums. sum = fma(w, s, sum) and weight = weight + w round once per tap, each by at most half an ulp of the running
  value: delta_S <= sum_k hulp(S_k), delta_W <= sum_k hulp(W_k) in the kernel's tap order (rows of the disc top to
  bottom, left to right in a row). They move the quotient by (delta_S + v delta_W) / W.
- The approximate reciprocal of the weight (eps |v|) and the rounding of fma(rcp, sum, 0.5) (eps/2 (v + 0.5)).
The sum of the three, times 1.01, is `bound`: the u16 output is floor(v + 0.5) exactly where v + 0.5 is farther than
`bound` from an integer, and within 1 of it elsewhere.

Outlier fusion (cuda_depth_processing.cu:168-227 / :337-397). A non-zero filtered depth d at (x, y) unprojects to
p = d ((x - cx + 0.5) / fx, (y - cy + 0.5) / fy, 1); each other frame k maps it to o = M_k (p, 1); o_z <= 0 fails;
(u, v) = (o_x / o_z fx + cx, o_y / o_z fy + cy) truncates toward zero to a pixel, which fails outside the image or on
a zero depth s; otherwise the frame agrees when (1 - tol) o_z <= s <= (1 + tol) o_z. The pixel is kept when at least
`required` frames agree (all K for required -1), and then passes the filtered value through unchanged.
Error: p is off by at most 2 eps d g per coordinate with g = 1 + (|x| + |cx| + 1) / |fx| + (|y| + |cy| + 1) / |fy|
(the fp32 unprojection constants, one fma and one product); one row of M (p, 1) adds four roundings of its running
value, so o is within 2 eps (sum_j |m_j p_j| + |m_3| + (|m_0| + |m_1|) d g) per coordinate; the approximate
reciprocal of o_z, the product and the fma of the projection add 1.5 eps |o_x / o_z| |fx| + eps/2 |u|. The margins
below are twice these. A frame's decision is exact unless o_z is within its margin of 0, u or v is within its margin
of a non-zero integer (truncation maps (-1, 1) to 0, so 0 is not an edge), or s is within its margin of
(1 +- tol) o_z (the fp32 1 +- tol and its product add eps |o_z|). A pixel's keep / drop is exact when it is the same
for every resolution of its inexact frames.

Erosion, the copy without border (radius 0), the four-neighbour rule of the normals stage and the count of 8
neighbours of the radii stage are integer work and restated exactly. Normals and radii themselves are held to
`normals64` / `radii64` of tests/test_camera_geometry_gpu.py.
"""
import numpy as np

EPS = 2.0 ** -23
LOG2E = 1.4426950408889634
FLUSH = -126.0   # ex2 arguments below this flush to zero


def f32(v):
    return float(np.float32(v))


def bilateral_radius(sigma_xy, radius_factor):
    """R = int(radius_factor * sigma_xy + 0.5f) in fp32, as the host computes it."""
    return int(np.float32(np.float32(radius_factor) * np.float32(sigma_xy)) + np.float32(0.5))


def valid_region(width, height, radius):
    """Pixels whose fp32 u32 squared distance to (W / 2, H / 2) is at most the fp32 radius^2."""
    y, x = np.mgrid[0:height, 0:width].astype(np.int64)
    d2 = ((x - width // 2) ** 2 + (y - height // 2) ** 2) % (1 << 32)
    r = np.float32(radius)
    return d2.astype(np.float32) <= np.float32(r * r)


def _hulp(x):
    """Half an fp32 ulp of the fp32 neighbour of x > 0 (x raised by 2^-10 covers a partial sum that is on the other
    side of a power of two in fp32); 0 for x == 0."""
    _, e = np.frexp(x * (1 + 2.0 ** -10))
    return np.where(x > 0, np.ldexp(1.0, e - 25), 0.0)


def disc_taps(R):
    return [(dy, dx) for dy in range(-R, R + 1) for dx in range(-R, R + 1) if dx * dx + dy * dy <= R * R]


class Bilateral:
    """value (float64 v, NaN where the output is value_to_ignore), active (v is defined), bound, expected (the
    u16 output where it is exact), clear (the output is exact) and the tap count of every pixel."""

    def __init__(self, raw, sigma_xy, sigma_value_factor, radius_factor, max_depth, valid_radius, value_to_ignore=0):
        raw = np.asarray(raw)
        H, W = raw.shape
        self.R = R = bilateral_radius(sigma_xy, radius_factor)
        sxy, sv = f32(sigma_xy), f32(sigma_value_factor)
        ignore = int(value_to_ignore)
        c = raw.astype(np.float64)
        self.active = valid_region(W, H, valid_radius) & (raw != ignore) & (raw <= int(max_depth))
        pad = np.full((H + 2 * R, W + 2 * R), ignore, np.int64)
        pad[R:R + H, R:R + W] = raw
        csafe = np.where(c > 0, c, 1.0)
        denom_v = 2 * (csafe * sv) ** 2

        def tap(dy, dx):
            s = pad[R + dy:R + dy + H, R + dx:R + dx + W]
            use = (s != ignore) & self.active
            u = -(dx * dx + dy * dy) / (2 * sxy * sxy) - (c - s) ** 2 / denom_v
            return s.astype(np.float64), use, np.where(use, np.exp(u), 0.0), u

        S, Wt, dS, dW = (np.zeros((H, W)) for _ in range(4))
        self.taps = np.zeros((H, W), np.int32)
        taps = disc_taps(R)
        for dy, dx in taps:
            s, use, w, _ = tap(dy, dx)
            S += w * s
            Wt += w
            dS += np.where(use, _hulp(S), 0.0)
            dW += np.where(use, _hulp(Wt), 0.0)
            self.taps += use
        Wsafe = np.where(self.active, Wt, 1.0)
        v = S / Wsafe
        P = np.zeros((H, W))
        for dy, dx in taps:
            s, use, w, u = tap(dy, dx)
            eta = np.where(u * LOG2E < FLUSH + 1, 1.0, 5 * EPS * np.abs(u) + 4 * EPS)
            P += np.where(use, w * eta * np.abs(s - v), 0.0)
        P /= Wsafe
        quotient = 1.001 * (dS + (v + P) * dW) / Wsafe
        bound = 1.01 * (1.001 * P + quotient + EPS * v + EPS / 2 * (v + 1.5))
        self.value = np.where(self.active, v, np.nan)
        self.bound = np.where(self.active, bound, 0.0)
        half = v + 0.5
        self.expected = np.where(self.active, np.floor(half), ignore).astype(np.int64)
        self.clear = ~self.active | (np.abs(half - np.round(half)) > bound)
        self.ignore = ignore

    def check(self, out):
        """(violations, fraction of the bound the worst pixel uses, share of active pixels inside the margin).
        A violation is an inexact output on a clear pixel, or an output farther than `bound` allows."""
        out = np.asarray(out).astype(np.int64)
        wrong_clear = int(((out != self.expected) & self.clear).sum())
        # the kernel value consistent with `out` lies in [out - 0.5, out + 0.5): its least distance to v
        v = np.where(self.active, self.value, 0.0)
        dev = np.maximum(np.maximum(out - 0.5 - v, v - (out + 0.5)), 0.0)
        frac = np.where(self.active, dev / np.where(self.bound > 0, self.bound, 1.0), 0.0)
        beyond = int((self.active & (dev > self.bound)).sum()) + int(((out != self.ignore) & ~self.active).sum())
        share = float((self.active & ~self.clear).sum() / max(int(self.active.sum()), 1))
        return wrong_clear + beyond, float(frac.max(initial=0.0)), share


class Outlier:
    """keep (float64 decision), clear (the decision is exact), ok_lo / ok_hi (agreeing frames, certain / possible)."""

    def __init__(self, depth, cam, others, mats, tolerance, required=-1):
        depth = np.asarray(depth)
        W, H, fx, fy, cx, cy = cam
        fx, fy, cx, cy, tol = f32(fx), f32(fy), f32(cx), f32(cy), f32(tolerance)
        mats = np.asarray(mats, np.float32).reshape(-1, 3, 4).astype(np.float64)
        K = len(others)
        assert mats.shape[0] == K
        y, x = np.mgrid[0:H, 0:W].astype(np.float64)
        d = depth.astype(np.float64)
        p = np.stack([d * (x - (cx - 0.5)) / fx, d * (y - (cy - 0.5)) / fy, d])
        g = 1 + (np.abs(x) + abs(cx) + 1) / abs(fx) + (np.abs(y) + abs(cy) + 1) / abs(fy)
        dp = 2 * EPS * d * g
        lo = np.zeros((H, W), np.int32)
        hi = np.zeros((H, W), np.int32)
        for k in range(K):
            m = mats[k]
            o = np.einsum("ij,jhw->ihw", m[:, :3], p) + m[:, 3][:, None, None]
            mag = np.einsum("ij,jhw->ihw", np.abs(m[:, :3]), np.abs(p)) + np.abs(m[:, 3])[:, None, None]
            do = 2 * 2 * EPS * (mag + (np.abs(m[:, 0]) + np.abs(m[:, 1]))[:, None, None] * d * g)
            ox, oy, oz = o
            front = oz > do[2]
            maybe_front = oz > -do[2]
            zs = np.where(np.abs(oz) > 0, np.abs(oz), 1.0)
            uu, vv = ox / zs * np.sign(oz) * fx + cx, oy / zs * np.sign(oz) * fy + cy
            du = 2 * (abs(fx) * (do[0] + np.abs(ox / zs) * do[2]) / zs + 1.5 * EPS * np.abs(ox / zs) * abs(fx)
                      + EPS / 2 * np.abs(uu))
            dv = 2 * (abs(fy) * (do[1] + np.abs(oy / zs) * do[2]) / zs + 1.5 * EPS * np.abs(oy / zs) * abs(fy)
                      + EPS / 2 * np.abs(vv))
            near_edge = (_near_nonzero_integer(uu, du) | _near_nonzero_integer(vv, dv))
            ix, iy = np.trunc(uu), np.trunc(vv)
            inside = (ix >= 0) & (iy >= 0) & (ix < W) & (iy < H)
            s = np.asarray(others[k])[np.clip(iy, 0, H - 1).astype(np.int64), np.clip(ix, 0, W - 1).astype(np.int64)]
            s = s.astype(np.float64)
            upper, lower = (1 + tol) * oz, (1 - tol) * oz
            dtol = (1 + tol) * do[2] + EPS * (1 + tol) * np.abs(oz)
            agree = front & inside & (s != 0) & (s <= upper) & (s >= lower)
            exact = (front | ~maybe_front) & ~near_edge & (np.abs(s - upper) > dtol) & (np.abs(s - lower) > dtol)
            lo += agree & exact
            hi += agree | ~exact
        req = K if required == -1 else required
        live = depth != 0
        self.keep = live & (lo >= req)
        self.clear = ~live | ((lo >= req) == (hi >= req))
        self.ok_lo, self.ok_hi = lo, hi

    def check(self, filtered, out):
        """(wrong decisions on clear pixels, share of live pixels inside a margin). Every output is 0 or the
        filtered value; kept pixels pass it through unchanged."""
        filtered, out = np.asarray(filtered), np.asarray(out)
        assert ((out == 0) | (out == filtered)).all(), "an output is neither 0 nor the filtered value"
        kept = out != 0
        wrong = int(((kept != self.keep) & self.clear).sum())
        live = filtered != 0
        return wrong, float((live & ~self.clear).sum() / max(int(live.sum()), 1))


def _near_nonzero_integer(u, margin):
    n = np.round(u)
    n = np.where(n == 0, np.where(u >= 0, 1.0, -1.0), n)
    return np.abs(u - n) <= margin


def erode64(depth, radius):
    """ErodeDepthMapCUDA / CopyWithoutBorderCUDA: a pixel survives when it is at least `radius` (1 for radius 0)
    from every border and its (2 radius + 1)^2 window has no zero."""
    depth = np.asarray(depth)
    H, W = depth.shape
    out = np.zeros_like(depth)
    r = max(radius, 1)
    if H <= 2 * r or W <= 2 * r:
        return out
    if radius == 0:
        out[1:-1, 1:-1] = depth[1:-1, 1:-1]
        return out
    ok = np.ones((H - 2 * r, W - 2 * r), bool)
    for dy in range(2 * r + 1):
        for dx in range(2 * r + 1):
            ok &= depth[dy:dy + H - 2 * r, dx:dx + W - 2 * r] != 0
    out[r:H - r, r:W - r] = np.where(ok, depth[r:H - r, r:W - r], 0)
    return out


def four_neighbours(depth):
    """Pixels whose centre and four neighbours are non-zero (zero outside the image)."""
    d = np.pad(np.asarray(depth) != 0, 1)
    return d[1:-1, 1:-1] & d[1:-1, :-2] & d[1:-1, 2:] & d[:-2, 1:-1] & d[2:, 1:-1]


def neighbour_count(depth):
    """Non-zero pixels among the eight neighbours (zero outside the image)."""
    d = np.pad(np.asarray(depth) != 0, 1).astype(np.int32)
    H, W = np.asarray(depth).shape
    return sum(d[1 + dy:1 + dy + H, 1 + dx:1 + dx + W] for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dy or dx)


def ignored_taps_vanish(sigma_value_factor, value_to_ignore=0):
    """The host's choice of the fused bilateral instantiation that drops the value_to_ignore test: 1 / (2 s^2) > 110
    in fp32 (an ignored tap's weight then flushes to zero)."""
    s = np.float32(sigma_value_factor)
    return value_to_ignore == 0 and s > 0 and np.float32(1.0) / np.float32(np.float32(2.0) * s * s) > np.float32(110.0)
