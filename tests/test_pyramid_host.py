"""Host-side checks of the --pyramid_level input downscaling (APP/main.cc:299-303, 946-981): the plain-C
restatement (tests/pyramid_walk.c) against a line-by-line Python port of the reference's libvis loops, the
scaled camera against libvis Camera::Scaled, and the argument checks of the two C entry points (they return
before touching the device)."""
import ctypes as C

import numpy as np
import pytest

from surfelmeshing_b200 import _lib
from surfelmeshing_b200.synthetic import Camera
from tests import pyramid_walk


def libvis_downscale_median(image, value_to_ignore, output_width, output_height):
    """Image<u16>::DownscaleUsingMedianWhileExcluding (libvis image.h:1003-1050), loop for loop: std::sort,
    float sum, `fabs(average - low) < fabs(average - high)`."""
    height, width = image.shape
    out = np.empty((output_height, output_width), dtype=np.uint16)
    for y in range(output_height):
        for x in range(output_width):
            start_x, end_x = (width * x) // output_width, (width * (x + 1)) // output_width
            start_y, end_y = (height * y) // output_height, (height * (y + 1)) // output_height
            values = []
            value_sum = np.float32(0)
            for original_y in range(start_y, end_y):
                for original_x in range(start_x, end_x):
                    value = int(image[original_y, original_x])
                    if value != value_to_ignore:
                        values.append(value)
                        value_sum = np.float32(value_sum + np.float32(value))
            if not values:
                out[y, x] = value_to_ignore
                continue
            average = np.float32(value_sum / np.float32(len(values)))
            values.sort()
            if len(values) % 2 == 1:
                out[y, x] = values[len(values) // 2]
            else:
                low, high = values[len(values) // 2 - 1], values[len(values) // 2]
                out[y, x] = low if abs(average - np.float32(low)) < abs(average - np.float32(high)) else high
    return out


def libvis_downscale_to_half_size(image):
    """Image<Vec3u8>::DownscaleToHalfSize (libvis image.h:929-948): a/4 + b/4 + c/4 + d/4, each quarter truncated."""
    height, width = image.shape[:2]
    assert width % 2 == 0 and height % 2 == 0
    v = image.astype(np.int32)
    return (v[0::2, 0::2] // 4 + v[0::2, 1::2] // 4 + v[1::2, 0::2] // 4 + v[1::2, 1::2] // 4).astype(np.uint8)


def libvis_image_pyramid(image, level):
    for _ in range(level):
        image = libvis_downscale_to_half_size(image)
    return image


def depth_case(shape, seed, value_to_ignore=0):
    """Close values (the even-count rule decides), holes, whole ignored blocks and the largest u16."""
    H, W = shape
    rng = np.random.RandomState(seed)
    depth = (3000 + rng.randint(0, 4, size=(H, W))).astype(np.uint16)
    far = rng.rand(H, W) < 0.2
    depth[far] = rng.randint(0, 65536, size=int(far.sum()))
    depth[rng.rand(H, W) < 0.3] = value_to_ignore
    depth[: H // 4, : W // 4] = value_to_ignore         # blocks with nothing left
    depth[rng.rand(H, W) < 0.05] = 65535
    return depth


@pytest.mark.parametrize("in_shape,out_shape", [
    ((8, 8), (4, 4)), ((6, 10), (3, 5)), ((16, 12), (4, 3)), ((5, 7), (2, 3)), ((7, 9), (7, 9)),
    ((201, 333), (67, 111)), ((48, 64), (3, 4)), ((45, 61), (4, 5)), ((33, 17), (6, 2))])
@pytest.mark.parametrize("value_to_ignore", [0, 3001])
def test_depth_restatement_matches_libvis_loop(in_shape, out_shape, value_to_ignore):
    depth = depth_case(in_shape, sum(in_shape) + value_to_ignore, value_to_ignore)
    H, W = out_shape
    expect = libvis_downscale_median(depth, value_to_ignore, W, H)
    got = pyramid_walk.downscale_median_excluding(depth, W, H, value_to_ignore)
    assert np.array_equal(got, expect)


def test_depth_even_count_rule_and_extremes():
    """Hand-made 2 x 2 blocks: the even-count rule picks the middle value closer to the float average (the
    upper one on a tie), ignored values are dropped and an all-ignored block gives value_to_ignore."""
    blocks = {
        (1, 2, 3, 100): 3,          # average 26.5: 3 is closer than 2? |26.5-2| > |26.5-3| -> upper 3
        (1, 2, 3, 4): 3,            # average 2.5: tie -> upper
        (10, 10, 11, 50): 11,       # average 20.25: 11 is closer than 10
        (0, 5, 6, 0): 6,            # two values left, average 5.5: tie -> upper
        (0, 0, 0, 0): 0,            # nothing left
        (0, 7, 0, 0): 7,            # one value
        (65535, 65535, 65534, 0): 65535,
        (1, 1, 2, 65535): 2,        # average 16384.75: upper
        (1, 100, 101, 102): 100,    # average 76: 100 closer than 101? |76-100| < |76-101| -> lower 100
    }
    keys = list(blocks)
    depth = np.zeros((2, 2 * len(keys)), dtype=np.uint16)
    for i, (a, b, c, d) in enumerate(keys):
        depth[:, 2 * i: 2 * i + 2] = [[a, b], [c, d]]
    expect = np.array([blocks[k] for k in keys], dtype=np.uint16)[None]
    assert np.array_equal(libvis_downscale_median(depth, 0, len(keys), 1), expect)
    assert np.array_equal(pyramid_walk.downscale_median_excluding(depth, len(keys), 1), expect)


@pytest.mark.parametrize("shape", [(2, 2), (4, 6), (16, 16), (48, 64), (32, 80)])
@pytest.mark.parametrize("level", [0, 1, 2, 3, 4])
def test_color_restatement_matches_libvis_loop(shape, level):
    H, W = shape
    if H % (1 << level) or W % (1 << level):
        pytest.skip("odd size at some level")
    rng = np.random.RandomState(H * W + level)
    color = rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8)
    color[0, :, 0] = 255
    assert np.array_equal(pyramid_walk.color_image_pyramid(color, level), libvis_image_pyramid(color, level))


def test_color_truncation_quirk():
    """Each quarter is truncated before the sum (the reference's own TODO, image.h:940): (1, 1, 2, 2) gives 0,
    not 1, and two levels are not one 4 x 4 average."""
    block = np.array([[1, 1], [2, 2]], dtype=np.uint8)
    color = np.repeat(block[:, :, None], 3, axis=2)
    assert pyramid_walk.color_image_pyramid(color, 1).tolist() == [[[0, 0, 0]]]
    color = np.full((4, 4, 3), 7, dtype=np.uint8)   # level 1: 1+1+1+1 = 4; level 2: 1+1+1+1 = 4
    assert pyramid_walk.color_image_pyramid(color, 2).tolist() == [[[4, 4, 4]]]
    assert int(color.astype(np.int32).mean()) == 7


@pytest.mark.parametrize("size", [(640, 480), (1280, 960), (641, 481)])
@pytest.mark.parametrize("level", [1, 2, 3])
def test_camera_scaled_matches_libvis(size, level):
    """Camera::Scaled(1 / 2^L) (libvis camera.h:1564-1573; APP/main.cc:751): the float factor 1.0f / powf(2, L);
    sizes int(factor * size + 0.5) in double; fx, fy, cx, cy (pixel corner) times the factor in float."""
    cam = Camera.tum(*size)
    scaled = cam.scaled(level)
    factor = np.float32(1.0) / np.float32(2.0 ** level)
    assert (scaled.width, scaled.height) == (int(float(factor) * size[0] + 0.5), int(float(factor) * size[1] + 0.5))
    for name in ("fx", "fy", "cx", "cy"):
        assert np.float32(getattr(scaled, name)) == np.float32(np.float32(getattr(cam, name)) * factor), name
    if size[0] % (1 << level) == 0:
        assert (scaled.width, scaled.height) == (size[0] >> level, size[1] >> level)
        assert scaled == Camera.tum(size[0] >> level, size[1] >> level)


def test_camera_scaled_known_values():
    assert Camera.tum(640, 480).scaled(1) == Camera(320, 240, 262.5, 262.5, 160.0, 120.0)
    assert Camera.tum(1280, 960).scaled(3) == Camera(160, 120, 131.25, 131.25, 80.0, 60.0)
    assert Camera.tum(640, 480).scaled(3) == Camera(80, 60, 65.625, 65.625, 40.0, 30.0)


def test_entry_points_reject_bad_arguments(product):
    """Size checks come first, so they need no device: every case is SM_ERR_INVALID_ARGUMENT."""
    depth = product.fn["downscale_using_median_while_excluding"]
    bad_depth = [
        (640, 480, 0, 240),      # empty output
        (640, 480, 320, 0),
        (640, 480, 641, 480),    # larger than the input
        (640, 480, 640, 481),
        (340, 480, 20, 480),     # 17 pixels wide blocks
        (640, 480, 640, 28),     # 18 rows
        (0, 480, 1, 1),
        (640, 480, 320, 240),    # valid sizes, null buffers
    ]
    for in_w, in_h, out_w, out_h in bad_depth:
        status = depth(None, 0, in_w, in_h, None, 2 * max(in_w, 1), out_w, out_h, None, 2 * max(out_w, 1))
        assert status == _lib.SM_ERR_INVALID_ARGUMENT, (in_w, in_h, out_w, out_h)
    color = product.fn["color_image_pyramid"]
    bad_color = [
        (-1, 640, 480), (5, 640, 480),   # levels outside [0, 4]
        (2, 642, 480),                   # 321 is odd at level 1
        (1, 640, 481),
        (4, 640, 488),                   # 61 is odd at level 3
        (1, 0, 480),
        (1, 640, 480),                   # valid sizes, null buffers
    ]
    for levels, w, h in bad_color:
        status = color(None, levels, w, h, None, 3 * max(w, 1), None, 3 * max(w, 1))
        assert status == _lib.SM_ERR_INVALID_ARGUMENT, (levels, w, h)
    assert product.fn["last_error"]()
