"""GPU checks of the --pyramid_level input downscaling (APP/main.cc:299-303, 946-981): the two kernels bit for
bit against the plain-C restatement (tests/pyramid_walk.c), sm_stream_run with pyramid_level against the same
run on frames downscaled beforehand, against the reference's kernels fed host-downscaled frames (main.cc's
path), and the argument checks of the stream runner."""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, SurfelError
from tests import pyramid_walk
from tests.test_pyramid_host import depth_case
from tests.util import count_mismatch

pytestmark = pytest.mark.gpu

# SoA rows compared exactly after one frame: positions, confidence, radius, normals, stamps (the smooth rows
# are left out: the regularisation sums with float atomics)
EXACT_ROWS = (0, 1, 2, 6, 7, 8, 9, 10, 17, 18)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make(cam, cap=400_000, lib=None):
    return R.CUDASurfelReconstruction(cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=lib)


# ---------------------------------------------------------------------------------------
# the two kernels
# ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("in_shape,out_shape", [
    ((480, 640), (240, 320)), ((480, 640), (120, 160)), ((480, 640), (60, 80)), ((960, 1280), (480, 640)),
    ((201, 333), (67, 111)), ((5, 7), (2, 3)),
    ((480, 640), (30, 40)), ((201, 333), (15, 25)), ((45, 61), (4, 5))])   # the last three: 9 to 16 pixel blocks
def test_downscale_depth_bit_exact(product, in_shape, out_shape):
    depth = depth_case(in_shape, in_shape[0] + out_shape[0])
    expect = pyramid_walk.downscale_median_excluding(depth, out_shape[1], out_shape[0])
    got = R.DownscaleUsingMedianWhileExcluding(None, 0, out_shape[1], out_shape[0], dev(depth), lib=product)
    torch.cuda.synchronize()
    assert count_mismatch(got.cpu().numpy(), expect) == 0


@pytest.mark.parametrize("value_to_ignore", [0, 3001])
def test_downscale_depth_pitched(product, value_to_ignore):
    """Input and output rows wider than the image; a value_to_ignore other than 0."""
    depth = depth_case((96, 128), 5, value_to_ignore)
    src = torch.full((96, 128 + 40), 1234, dtype=torch.uint16, device="cuda")
    src[:, :128] = dev(depth)
    for out_h, out_w in ((48, 64), (24, 32), (8, 10)):
        out = torch.full((out_h, out_w + 24), 4321, dtype=torch.uint16, device="cuda")
        R.DownscaleUsingMedianWhileExcluding(None, value_to_ignore, out_w, out_h, src[:, :128], out[:, :out_w],
                                             lib=product)
        torch.cuda.synchronize()
        expect = pyramid_walk.downscale_median_excluding(depth, out_w, out_h, value_to_ignore)
        assert count_mismatch(out[:, :out_w].cpu().numpy(), expect) == 0
        assert (out[:, out_w:] == 4321).all(), "nothing is written past the row"


@pytest.mark.parametrize("level", [0, 1, 2, 3, 4])
def test_color_pyramid_bit_exact(product, level):
    rng = np.random.RandomState(40 + level)
    color = rng.randint(0, 256, size=(480, 640, 3)).astype(np.uint8)
    expect = pyramid_walk.color_image_pyramid(color, level)
    got = R.ImagePyramid(None, dev(color), level, lib=product)
    torch.cuda.synchronize()
    assert np.array_equal(got.cpu().numpy(), expect)


def test_color_pyramid_pitched(product):
    rng = np.random.RandomState(3)
    color = rng.randint(0, 256, size=(96, 128, 3)).astype(np.uint8)
    src = torch.zeros((96, 128 + 16, 3), dtype=torch.uint8, device="cuda")
    src[:, :128] = dev(color)
    for level in (1, 2, 3):
        h, w = 96 >> level, 128 >> level
        out = torch.full((h, w + 8, 3), 77, dtype=torch.uint8, device="cuda")
        R.ImagePyramid(None, src[:, :128], level, output=out[:, :w], lib=product)
        torch.cuda.synchronize()
        assert np.array_equal(out[:, :w].cpu().numpy(), pyramid_walk.color_image_pyramid(color, level))
        assert (out[:, w:] == 77).all()


# ---------------------------------------------------------------------------------------
# sm_stream_run with pyramid_level
# ---------------------------------------------------------------------------------------

def pyramid_inputs(frames, stream_id, level=1, size=(640, 480)):
    """Full-size stream, the scaled camera and the frames downscaled beforehand by the standalone calls."""
    full = S.Camera.tum(*size)
    cam = full.scaled(level)
    st = S.make_stream(full, frames, stream_id=stream_id, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    small_depth = torch.stack([R.DownscaleUsingMedianWhileExcluding(None, 0, cam.width, cam.height, st.depth[i])
                               for i in range(frames)])
    small_color = torch.stack([R.ImagePyramid(None, st.color[i], level) for i in range(frames)])
    torch.cuda.synchronize()
    return cam, st, small_depth, small_color, pp, IntegrateParams.defaults()


def run(rec, st, depth, color, pp, ip, first, last):
    return rec.stream_run(None, depth, color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                          first, last)


def frames_for(st, on_host):
    if on_host:
        return st.depth.cpu().pin_memory(), st.color.cpu().pin_memory()
    return st.depth, st.color


def full_size_upload_bytes(st, first, last):
    """Every raw depth map of [first - K/2, last + K/2) and the colour images of [first, last), full-size."""
    F, H, W = st.depth.shape
    half = st.other_count // 2
    return (min(last + half, F) - max(first - half, 0)) * H * W * 2 + (last - first) * H * W * 3


@pytest.mark.parametrize("on_host", [False, True])
def test_one_frame_equals_downscaled_beforehand(product, on_host):
    cam, st, small_depth, small_color, pp, ip = pyramid_inputs(9, 21)
    first, last = 4, 5
    ref = make(cam)
    s0 = run(ref, st, small_depth, small_color, pp, ip, first, last)
    rec = make(cam)
    rec.configure("pyramid_level", 1)
    depth, color = frames_for(st, on_host)
    s1 = run(rec, st, depth, color, pp, ip, first, last)
    assert s1.frames_integrated == 1 and s1.surfels_size > 5_000
    assert s1.surfels_size == s0.surfels_size
    assert s1.h2d_bytes == (full_size_upload_bytes(st, first, last) if on_host else 0)
    assert np.array_equal(rec.download_rasters()["new_surfel_flag_vector"], ref.download_rasters()["new_surfel_flag_vector"])
    rows1, rows0 = rec.dump_state()[0], ref.dump_state()[0]
    for row in EXACT_ROWS:
        assert count_mismatch(rows1[row], rows0[row]) == 0, row


def test_stream_equals_downscaled_beforehand(product):
    cam, st, small_depth, small_color, pp, ip = pyramid_inputs(20, 22)
    first, last = st.integrated_range()
    s0 = run(make(cam), st, small_depth, small_color, pp, ip, first, last)
    assert s0.surfels_size > 10_000
    for on_host in (False, True):
        rec = make(cam)
        rec.configure("pyramid_level", 1)
        depth, color = frames_for(st, on_host)
        s1 = run(rec, st, depth, color, pp, ip, first, last)
        assert s1.frames_integrated == last - first
        assert abs(int(s1.surfels_size) - int(s0.surfels_size)) <= 0.002 * s0.surfels_size + 5
        assert abs(int(s1.surfel_count) - int(s0.surfel_count)) <= 0.002 * s0.surfel_count + 5
        assert s1.h2d_bytes == (full_size_upload_bytes(st, first, last) if on_host else 0)


def test_stream_against_reference(product, reference):
    """main.cc's path on the reference's kernels (frames downscaled on the host, scaled camera) against the
    product's pyramid_level = 1 on the full-size frames."""
    cam, st, small_depth, small_color, pp, ip = pyramid_inputs(20, 23)
    first, last = st.integrated_range()
    host_depth = np.stack([pyramid_walk.downscale_median_excluding(d, cam.width, cam.height) for d in st.depth.cpu().numpy()])
    host_color = np.stack([pyramid_walk.color_image_pyramid(c, 1) for c in st.color.cpu().numpy()])
    assert np.array_equal(host_depth, small_depth.cpu().numpy()) and np.array_equal(host_color, small_color.cpu().numpy())
    s_ref = run(make(cam, lib=reference), st, dev(host_depth), dev(host_color), pp, ip, first, last)
    rec = make(cam)
    rec.configure("pyramid_level", 1)
    s = run(rec, st, st.depth, st.color, pp, ip, first, last)
    assert abs(int(s.surfels_size) - int(s_ref.surfels_size)) <= max(5, 0.01 * s_ref.surfels_size), \
        (s.surfels_size, s_ref.surfels_size)


def expect_invalid(call):
    with pytest.raises(SurfelError) as e:
        call()
    assert e.value.code == _lib.SM_ERR_INVALID_ARGUMENT


def test_invalid_configurations_leave_the_handle_working(product):
    cam, st, small_depth, small_color, pp, ip = pyramid_inputs(9, 24)
    first, last = 4, 5
    rec = make(cam)
    for value in (5, 1.5, -1):
        expect_invalid(lambda: rec.configure("pyramid_level", value))
    # with median densify, in either configure order (main.cc:946-949)
    rec.configure("pyramid_level", 1)
    rec.configure("median_filter_and_densify_iterations", 1)
    expect_invalid(lambda: run(rec, st, st.depth, st.color, pp, ip, first, last))
    rec.configure("pyramid_level", 0)
    rec.configure("median_filter_and_densify_iterations", 1)
    rec.configure("pyramid_level", 1)
    expect_invalid(lambda: run(rec, st, st.depth, st.color, pp, ip, first, last))
    rec.configure("median_filter_and_densify_iterations", 0)
    # a width not divisible by 2^L
    odd_depth, odd_color = st.depth[:, :, :639].contiguous(), st.color[:, :, :639].contiguous()
    expect_invalid(lambda: run(rec, st, odd_depth, odd_color, pp, ip, first, last))
    # frames of the wrong size for the handle: 640 x 480 at level 2 is 160 x 120, the handle is 320 x 240
    rec.configure("pyramid_level", 2)
    expect_invalid(lambda: run(rec, st, st.depth, st.color, pp, ip, first, last))
    # and at level 0 the full-size frames do not fit either
    rec.configure("pyramid_level", 0)
    expect_invalid(lambda: run(rec, st, st.depth, st.color, pp, ip, first, last))
    # the handle still works, and a pyramid run on it equals one on a fresh handle
    rec.configure("pyramid_level", 1)
    s = run(rec, st, st.depth, st.color, pp, ip, first, last)
    fresh = make(cam)
    fresh.configure("pyramid_level", 1)
    s_fresh = run(fresh, st, st.depth, st.color, pp, ip, first, last)
    assert s.frames_integrated == 1 and s.surfels_size == s_fresh.surfels_size > 5_000
    rec.configure("pyramid_level", 0)
    s0 = run(make(cam), st, small_depth, small_color, pp, ip, first, last)
    rec.reset()
    assert run(rec, st, small_depth, small_color, pp, ip, first, last).surfels_size == s0.surfels_size
