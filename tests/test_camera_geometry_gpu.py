"""Float64 anchors of the closed-form stages on the cameras of real datasets, independent of the reference.

The parity tests compare the product with the reference through the same Python wrappers, so a mistake the two
share (an argument order, an fx / fy or cx / cy mix-up on the way in) passes them. Here the normals, the radii and the
surfels of a first Integrate() are restated in numpy float64 from the same u16 depths and the fp32 intrinsics the
library receives, and held to bounds derived from the fp32 operation count (eps = 2^-23):

Unprojection. p = d (X, Y, 1) with X = x fx_inv + cx_inv (one fma on two rounded constants; cx_inv carries two
roundings) and d = depth * (1 / scale) (two roundings). Each coordinate is off by at most ~3.5 eps d g with
g = 1 + (|x| + |cx|) / |fx| + (|y| + |cy|) / |fy| (the terms of the fma can cancel), so a point is off by at most
~6 eps E, E = d g with d the largest depth involved.

Normals. a = right - left, b = top - bottom: |delta a| <= 2 * 6 eps E + eps/2 |a| with the rounding of the
difference (one fused product), same for b. n = a x b (one product + one fma per component) is then off by at most
12 eps E (|a| + |b|) + 3 eps |a||b|; normalising a vector perturbed by delta moves its direction by at most
2 |delta| / |n|, and the approximate sqrt / reciprocal and three products add ~4 eps. With
kappa = E (|a| + |b|) / |a x b| (|p| over the shorter difference, divided by the sine of their angle) and
|a||b| / |a x b| <= 2 kappa (|a|, |b| <= 2E), the normal is within (24 + 12 + 4) kappa eps = 40 kappa eps
(kappa >= 1/2). The observation-angle test v.n adds the approximate rsqrt of the view direction, its three roundings
and the fp32 threshold: 40 kappa eps + 16 eps.

Radii. A neighbour offset o is off by at most 12 eps E + eps/2 |o|, so |o|^2 by 2 |o| (12 eps E) + 2 eps |o|^2;
relative to the smallest offset that enters (the maximum and the clamp are both at least it), with kappa_r =
E / min |o| and the fp32 extension / clamp factors: 24 kappa_r eps + 4 eps <= 32 kappa_r eps.
"""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams
from tests.test_parity_gpu import LIVE_CAMERAS, run_stages, u16
from tests.test_session_gpu import assert_one_frame_equal, run_session
from tests.util import count_mismatch, other_frames

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23
CAMERAS = ["tum_fr1", "icl_nuim", "odd"]


def f32(v):
    return float(np.float32(v))


def camera_case(name, frames=9):
    cam, scale = LIVE_CAMERAS[name]
    st = S.make_stream(cam, frames, stream_id=31, depth_scaling=scale, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    pp.depth_scaling = scale
    return cam, st, pp


def stages(cam, st, pp, frame):
    """The product's five pre-processing stages on one frame (numpy outputs)."""
    others = [st.depth[f] for f in other_frames(frame, pp.outlier_filtering_frame_count)]
    o = run_stages(None, (cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy), pp, st.depth[frame], others,
                   st.others_TR_reference[frame])
    return {k: v.cpu().numpy() for k, v in o.items()}


class Unprojection:
    """float64 unprojection with the fp32 intrinsics the library gets (pixel-corner cx, cy)."""

    def __init__(self, cam, scale):
        self.fx, self.fy, self.cx, self.cy = f32(cam.fx), f32(cam.fy), f32(cam.cx), f32(cam.cy)
        self.scale = float(scale)

    def direction(self, x, y):
        return (x - (self.cx - 0.5)) / self.fx, (y - (self.cy - 0.5)) / self.fy

    def point(self, x, y, depth_u16):
        d = depth_u16.astype(np.float64) / self.scale
        X, Y = self.direction(x, y)
        return np.stack([d * X, d * Y, d])

    def spread(self, x, y, depth_u16):
        """E = d g of the error model in the module docstring."""
        g = 1 + (np.abs(x) + abs(self.cx)) / abs(self.fx) + (np.abs(y) + abs(self.cy)) / abs(self.fy)
        return depth_u16.astype(np.float64) / self.scale * g


def normals64(U, depth, threshold_deg):
    """float64 normals stage on the interior of `depth` (u16 [H, W]): (normal [3, h, w], keep, valid, bound, dot
    bound) with h, w = H - 2, W - 2."""
    H, W = depth.shape
    y, x = np.mgrid[1:H - 1, 1:W - 1].astype(np.float64)
    c, l, r = depth[1:-1, 1:-1], depth[1:-1, :-2], depth[1:-1, 2:]
    t, b = depth[:-2, 1:-1], depth[2:, 1:-1]
    valid = (c != 0) & (l != 0) & (r != 0) & (t != 0) & (b != 0)
    a = U.point(x + 1, y, r) - U.point(x - 1, y, l)
    bb = U.point(x, y - 1, t) - U.point(x, y + 1, b)
    n = np.cross(a, bb, axis=0)
    length = np.linalg.norm(n, axis=0)
    safe = np.where(length > 0, length, 1.0)
    n = n / safe * (-1.0 if U.fy < 0 else 1.0)
    X, Y = U.direction(x, y)
    v = np.stack([X, Y, np.ones_like(X)]) / np.sqrt(X * X + Y * Y + 1)
    dot = (v * n).sum(axis=0)
    keep = dot < -np.cos(np.pi / 180 * threshold_deg)
    E = U.spread(x + 1, y + 1, np.maximum(np.maximum(l, r), np.maximum(t, b)))
    kappa = E * (np.linalg.norm(a, axis=0) + np.linalg.norm(bb, axis=0)) / safe
    bound = 40 * kappa * EPS
    # the kernel's degenerate branch (|n| <= 1e-6) is not part of this anchor
    valid &= length > 2e-6
    return n, keep, valid, bound, bound + 16 * EPS, dot


@pytest.mark.parametrize("camera", CAMERAS)
def test_normals_stage_against_float64(product, camera):
    cam, st, pp = camera_case(camera)
    U = Unprojection(cam, pp.depth_scaling)
    o = stages(cam, st, pp, 4)
    n64, keep64, valid, bound, dot_bound, dot = normals64(U, o["erode"], pp.observation_angle_threshold_deg)
    kept = o["normals_depth"][1:-1, 1:-1] != 0
    normals = o["normals"][1:-1, 1:-1].transpose(2, 0, 1).astype(np.float64)
    assert valid.sum() > 0.1 * valid.size
    err = np.abs(normals - n64[:2]).max(axis=0)
    assert (err[valid] <= bound[valid]).all(), f"normal off by {float((err / bound)[valid].max()):.2f} x the bound"
    clear = valid & (np.abs(dot - (-np.cos(np.pi / 180 * pp.observation_angle_threshold_deg))) > dot_bound)
    assert count_mismatch(kept, keep64, clear) == 0, "keep / drop decisions"
    e = o["erode"]
    five = (e[1:-1, 1:-1] != 0) & (e[1:-1, :-2] != 0) & (e[1:-1, 2:] != 0) & (e[:-2, 1:-1] != 0) & (e[2:, 1:-1] != 0)
    assert not (kept & ~five).any(), "a pixel without its four neighbours was kept"
    assert kept.sum() > 0.5 * valid.sum(), "most measured pixels face the camera"
    print(f"{camera}: {int(valid.sum())} pixels, {int(kept.sum())} kept, worst normal error "
          f"{float((err / bound)[valid].max()):.3f} of the bound, median kappa {float(np.median(bound[valid] / 40 / EPS)):.1f}")


def radii64(U, depth, extension, clamp):
    """float64 radii stage: (radius^2, neighbour count, relative bound) for every pixel of the normals-stage depth."""
    H, W = depth.shape
    pad = np.zeros((H + 2, W + 2), depth.dtype)
    pad[1:-1, 1:-1] = depth
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    p = U.point(x, y, depth)
    largest, smallest = np.zeros((H, W)), np.full((H, W), np.inf)
    count = np.zeros((H, W), np.int32)
    deepest = depth.astype(np.int64)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx == 0 and dy == 0:
                continue
            nd = pad[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]
            has = nd != 0
            d2 = ((U.point(x + dx, y + dy, nd) - p) ** 2).sum(axis=0)
            largest = np.where(has, np.maximum(largest, d2), largest)
            smallest = np.where(has, np.minimum(smallest, d2), smallest)
            count += has
            deepest = np.maximum(deepest, nd)
    with np.errstate(invalid="ignore", over="ignore"):
        extended, clamped = largest * extension ** 2, smallest * (clamp ** 2 * 2.0)
    kappa = U.spread(x + 1, y + 1, deepest) / np.sqrt(np.where(count > 0, smallest, 1.0))
    return np.minimum(extended, clamped), count, 32 * kappa * EPS, clamped < extended


@pytest.mark.parametrize("camera", CAMERAS)
@pytest.mark.parametrize("clamp", [float("inf"), 1.2])
def test_radii_stage_against_float64(product, camera, clamp):
    cam, st, pp = camera_case(camera)
    pp.point_radius_clamp_factor = clamp
    U = Unprojection(cam, pp.depth_scaling)
    o = stages(cam, st, pp, 4)
    nd = o["normals_depth"]
    r2, count, rel, clamped = radii64(U, nd, f32(pp.point_radius_extension_factor), f32(clamp))
    written = (nd != 0) & (count > 0)
    got = o["radius"].astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        err = np.abs(got - r2) / r2
    assert (err[written] <= rel[written]).all(), f"radius^2 off by {float((err / rel)[written].max()):.2f} x the bound"
    assert np.array_equal(o["pre_depth"] != 0, (nd != 0) & (count >= 8)), "isolated pixels"
    assert clamped[written].any() == (clamp != float("inf")), "the clamp bites exactly when it is finite"
    print(f"{camera} clamp {clamp}: worst radius error {float((err / rel)[written].max()):.3f} of the bound")


@pytest.mark.parametrize("camera", CAMERAS)
def test_first_integrate_against_float64(product, camera):
    """First Integrate() on an empty cloud: one surfel per kept interior pixel at global_T_local * unproject(pixel)
    (no blending without surfels), with the pixel's normal rotated to the world and its radius."""
    cam, st, pp = camera_case(camera)
    U = Unprojection(cam, pp.depth_scaling)
    frame = 4
    o = stages(cam, st, pp, frame)
    ip = IntegrateParams.defaults()
    ip.depth_scaling = pp.depth_scaling
    rec = R.CUDASurfelReconstruction(400_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    d = torch.from_numpy(o["pre_depth"].astype(np.int32)).to(torch.uint16).cuda()
    normals, radius = torch.from_numpy(o["normals"]).cuda(), torch.from_numpy(o["radius"]).cuda()
    rec.integrate(None, frame, ip, d, normals, radius, st.color[frame], st.global_T_frame[frame], st.frame_T_global[frame])
    torch.cuda.synchronize()
    ras = rec.download_rasters()
    rows, n, _ = rec.dump_state()
    flags = ras["new_surfel_flag_vector"] != 0
    assert np.array_equal(flags, o["pre_depth"] != 0) and n == int(flags.sum()) > 1000
    ys, xs = np.nonzero(flags)
    idx = ras["new_surfel_indices"][ys, xs].astype(np.int64)
    assert np.array_equal(np.sort(idx), np.arange(n))
    T = st.global_T_frame[frame].astype(np.float64)
    Rm, t = T[:, :3], T[:, 3]
    depth = o["pre_depth"][ys, xs]
    g = Rm @ U.point(xs.astype(np.float64), ys.astype(np.float64), depth) + t[:, None]
    bound = 12 * EPS * (U.spread(xs, ys, depth) + np.linalg.norm(t))
    err = np.abs(rows[0:3, idx] - g).max(axis=0)
    assert (err <= bound).all(), f"position off by {float((err / bound).max()):.2f} x the bound"
    nxy = o["normals"][ys, xs].astype(np.float64).T
    nz = -np.sqrt(np.maximum(1 - (nxy ** 2).sum(axis=0), 0))
    gn = Rm @ np.concatenate([nxy, nz[None]])
    n_bound = EPS * (16 + 4 / np.maximum(np.abs(nz), 1e-3))
    n_err = np.abs(rows[8:11, idx] - gn).max(axis=0)
    assert (n_err <= n_bound).all(), f"normal off by {float((n_err / n_bound).max()):.2f} x the bound"
    assert count_mismatch(rows[7, idx], o["radius"][ys, xs]) == 0, "radius^2"
    assert (rows[6, idx] == 1.0).all() and (rows[17, idx].view(np.uint32) == frame).all()
    print(f"{camera}: {n} surfels, worst position error {float((err / bound).max()):.3f} of the bound")


@pytest.mark.parametrize("camera", ["odd", "icl_nuim"])
def test_one_frame_graph_serial_and_session(product, camera):
    """One integrated frame on an anisotropic odd-width camera and on a negative-fy camera: the frame graph, serial
    mode and a session give the same surfels (the graph's tiled copies run with a ragged tail at an odd width)."""
    cam, st, pp = camera_case(camera)
    ip = IntegrateParams.defaults()
    others = R.stream_outlier_filter_transforms(st.global_T_frame, st.frame_T_global, 8, st.depth_scaling)
    make = lambda: R.CUDASurfelReconstruction(400_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    graph, serial, session = make(), make(), make()
    run = lambda rec: rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, others, pp, ip, 4, 5)
    assert run(graph).frames_integrated == 1
    serial.enable_timings(True)
    run(serial)
    stats = run_session(session, st, 9, pp, ip, size=(cam.width, cam.height))
    assert stats.frames_integrated == 1
    assert_one_frame_equal(serial, graph)
    assert_one_frame_equal(session, graph)


def test_vis_depth_processing_shims_anisotropic(product, shimref):
    """The vis:: shims on the odd camera (fx != fy, off-centre principal point, odd size): the reference's host glue
    linked against the product's kernels gives the product's own pre-processing bit for bit."""
    cam, st, pp = camera_case("odd")
    outs = []
    for lib in (product, shimref):
        rec = R.CUDASurfelReconstruction(100_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=lib)
        frame = 4
        others = [st.depth[f] for f in other_frames(frame, pp.outlier_filtering_frame_count)]
        H, W = cam.height, cam.width
        d, n = u16(H, W), torch.zeros((H, W, 2), device="cuda")
        r = torch.full((H, W), float("nan"), device="cuda")
        rec.preprocess(None, pp, st.depth[frame], others, st.others_TR_reference[frame], d, n, r)
        torch.cuda.synchronize()
        outs.append([v.cpu().numpy() for v in (d, n, r)])
    assert outs[0][0].any()
    for a, b in zip(outs[0], outs[1]):
        assert count_mismatch(a, b) == 0
