"""sm_outlier_filter_transforms (host only, APP/main.cc:1039-1058)."""
import ctypes as C

import numpy as np
import pytest

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R

FRAMES = 500            # the trajectory of bench.py's 500-frame VGA stream (stream_id 0)
DEPTH_SCALING = 5000.0
EPS = 2.0 ** -24        # unit roundoff of float32


@pytest.fixture(scope="module")
def poses():
    p64 = S.trajectory(FRAMES, 0)
    return p64, p64.astype(np.float32), S.invert_poses(p64).astype(np.float32)


def scaled(m32, s):
    m = m32.astype(np.float64)
    m[..., 3] *= np.float64(np.float32(s))
    return m


def restated(g32, l32, frame, K, s):
    """The header's evaluation order in float64 numpy (no fused operations), rounded to float32 once."""
    half = K // 2
    others = [frame - (i + 1) for i in range(half)] + [frame + (i + 1) for i in range(half)]
    A = scaled(l32[others], s)          # [K, 3, 4]
    B = scaled(g32[frame], s)           # [3, 4]
    m = np.empty((K, 3, 4))
    for c in range(4):
        v = A[:, :, 0] * B[0, c] + A[:, :, 1] * B[1, c]
        v = v + A[:, :, 2] * B[2, c]
        if c == 3:
            v = v + A[:, :, 3]
        m[:, :, c] = v
    return m.astype(np.float32)


@pytest.mark.parametrize("K", [2, 4, 6, 8])
def test_bit_exact_against_restatement(product, poses, K):
    _, g32, l32 = poses
    for frame in range(K // 2, FRAMES - K // 2):
        got = R.outlier_filter_transforms(g32, l32, frame, K, DEPTH_SCALING, lib=product)
        want = restated(g32, l32, frame, K, DEPTH_SCALING)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"frame {frame}"


@pytest.mark.parametrize("K", [2, 4, 6, 8])
def test_matches_float64_harness(product, poses, K):
    """Against synthetic.others_TR_reference, which builds the transforms from the float64 poses with an explicit
    inverse. The library gets the poses rounded to float32: each entry of A (frame_T_global) and B (global_T_frame)
    carries a relative error <= EPS, so an entry of A . B moves by at most EPS (2 + EPS) sum_k |A_rk B_kc| (+ EPS
    |A_r3| for the translation column), and the final rounding adds EPS |m|. The float64 harness itself is exact to
    ~1e-12 of the magnitudes involved."""
    p64, g32, l32 = poses
    harness = S.others_TR_reference(p64, DEPTH_SCALING, K).astype(np.float64)
    half = K // 2
    for frame in range(half, FRAMES - half):
        got = R.outlier_filter_transforms(g32, l32, frame, K, DEPTH_SCALING, lib=product).astype(np.float64)
        others = [frame - (i + 1) for i in range(half)] + [frame + (i + 1) for i in range(half)]
        A = np.abs(scaled(l32[others], DEPTH_SCALING))
        B = np.abs(scaled(g32[frame], DEPTH_SCALING))
        products = A[:, :, :3] @ B   # sum_k |A_rk| |B_kc|
        translation = np.zeros_like(products)
        translation[:, :, 3] = A[:, :, 3]
        bound = EPS * ((2 + EPS) * products + translation + np.abs(harness[frame])) + 1e-12 * (products + translation)
        err = np.abs(got - harness[frame])
        assert np.all(err <= bound), f"frame {frame}: worst excess {np.max(err - bound):.3g}"


def test_rejections(product, poses):
    _, g32, l32 = poses
    out = np.zeros((8, 12), np.float32)
    call = lambda K, frame, n=FRAMES: product.fn["outlier_filter_transforms"](
        K, DEPTH_SCALING, n, g32.ctypes.data_as(C.c_void_p), l32.ctypes.data_as(C.c_void_p), frame,
        out.ctypes.data_as(C.c_void_p))
    for K in (0, 1, 3, 5, 7, 9, 10, -2):
        assert call(K, 100) == _lib.SM_ERR_INVALID_ARGUMENT, K
    for K in (2, 4, 6, 8):
        half = K // 2
        assert call(K, half) == _lib.SM_OK
        assert call(K, FRAMES - half - 1) == _lib.SM_OK
        assert call(K, half - 1) == _lib.SM_ERR_INVALID_ARGUMENT
        assert call(K, FRAMES - half) == _lib.SM_ERR_INVALID_ARGUMENT
        assert call(K, 12, n=12 + half) == _lib.SM_ERR_INVALID_ARGUMENT
    assert product.fn["outlier_filter_transforms"](8, DEPTH_SCALING, FRAMES, None, None, 100,
                                                   out.ctypes.data_as(C.c_void_p)) == _lib.SM_ERR_INVALID_ARGUMENT
    assert b"other_count" in product.fn["last_error"]() or b"null" in product.fn["last_error"]()


def test_stream_transforms_match_per_frame_call(product, poses):
    _, g32, l32 = poses
    allf = R.stream_outlier_filter_transforms(g32[:30], l32[:30], 8, DEPTH_SCALING, lib=product)
    assert allf.shape == (30, 8, 3, 4)
    assert np.array_equal(allf[10], R.outlier_filter_transforms(g32[:30], l32[:30], 10, 8, DEPTH_SCALING, lib=product))
    assert np.array_equal(allf[0], np.tile(np.eye(4, dtype=np.float32)[:3], (8, 1, 1)))
