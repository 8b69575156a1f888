"""sm_stream_run and sessions at a bilateral radius other than 6: the frame graph then runs k_bilateral_generic
and k_outlier in place of the fused radius-6 kernel, and must compute what the serial mode computes."""
import pytest

from surfelmeshing_b200 import _lib
from surfelmeshing_b200._lib import SurfelError
from tests.test_session_gpu import CAM, assert_one_frame_equal, make, near, run_session, run_stream, vga  # noqa: F401
from tests.util import params

pytestmark = pytest.mark.gpu


def radius4():
    """bilateral_filter_sigma_xy = 2 with the default radius factor 2: radius 4."""
    pp, ip = params(CAM)
    pp.bilateral_filter_sigma_xy = 2.0
    assert int(pp.bilateral_filter_radius_factor * pp.bilateral_filter_sigma_xy + 0.5) == 4
    return pp, ip


def test_graph_against_serial(product, vga):
    st, others = vga
    pp, ip = radius4()
    for n in (9, 60):
        graph, serial = make(), make()
        serial.enable_timings(True)
        got = run_stream(graph, st, others, n, pp, ip)
        want = run_stream(serial, st, others, n, pp, ip)
        assert got.frames_integrated == want.frames_integrated == n - 8
        if n == 9:
            assert_one_frame_equal(graph, serial)
        else:
            assert near(got.surfels_size, want.surfels_size) and near(got.surfel_count, want.surfel_count)


def test_session_against_stream(product, vga):
    st, others = vga
    pp, ip = radius4()
    ref = make()
    run_stream(ref, st, others, 9, pp, ip)
    rec = make()
    stats = run_session(rec, st, 9, pp, ip)
    assert stats.frames_integrated == 1
    assert_one_frame_equal(rec, ref)


def test_negative_radius_is_rejected(product, vga):
    st, others = vga
    pp, ip = params(CAM)
    rec = make()
    pp.bilateral_filter_sigma_xy = -3.0
    with pytest.raises(SurfelError) as err:
        run_stream(rec, st, others, 9, pp, ip)
    assert err.value.code == _lib.SM_ERR_INVALID_ARGUMENT
    pp, ip = params(CAM)
    assert run_stream(rec, st, others, 9, pp, ip).frames_integrated == 1
