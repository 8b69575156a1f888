"""The meta word of every regularisation record matches the surfel's stamp and detach flag.

The smooth positions live in 16-byte records {x, y, z, last_update_stamp | detach << 31}, double-buffered; the
regularisation sweeps read the stamp and the detach flag of a neighbour from its record. Every writer of a stamp
or of the colour's detach byte therefore has to write the meta word of BOTH buffers. sm_dump_state shows the
current buffer in rows 3-5 and 15; the other buffer becomes the current one at the next sweep, so a writer that
forgets one buffer shows up at a later check of this test."""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams
from tests.test_regularize_window_gpu import SEQUENCES, integrate

pytestmark = pytest.mark.gpu

STAMP_ROW = R.ROW_NAMES.index("last_update_stamp")
COLOR_ROW = R.ROW_NAMES.index("color")
META_ROW = R.ROW_NAMES.index("accum_y")
W, H = 320, 240


@pytest.fixture(scope="module")
def stream():
    cam = S.Camera.tum(W, H)
    st = S.make_stream(cam, 40, stream_id=3, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    torch.cuda.synchronize()
    return cam, st, pp


def check_meta(rec, where):
    rows, n, merges = rec.dump_state()
    stamps = rows[STAMP_ROW, :n].view(np.uint32)
    detach = (rows[COLOR_ROW, :n].view(np.uint32) >> np.uint32(24)) == np.uint32(1)
    expected = stamps | np.where(detach, np.uint32(0x80000000), np.uint32(0))
    meta = rows[META_ROW, :n].view(np.uint32)
    bad = np.flatnonzero(meta != expected)
    assert bad.size == 0, (f"{where}: {bad.size} of {n} slots with a stale meta word, first slot {bad[0]}: "
                           f"{meta[bad[0]]:#x} != {expected[bad[0]]:#x}")
    return n, merges, int(detach.sum())


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_meta_word_matches_stamp_and_detach_flag(product, stream, name):
    cam, st, pp = stream
    rec = R.CUDASurfelReconstruction(400_000, W, H, cam.fx, cam.fy, cam.cx, cam.cy)
    checked = merges = detached = 0
    try:
        for frame, frame_index, window, iterations, action in SEQUENCES[name]:
            if action == "reload":
                rows, _, merge_count = rec.dump_state()
                rec.load_state(rows, merge_count)
                check_meta(rec, f"load_state before frame {frame_index}")
            elif action == "reset":
                rec.reset()
            ip = IntegrateParams.defaults()
            ip.regularization_frame_window_size = window
            ip.regularization_iterations_per_integration_iteration = iterations
            integrate(rec, st, pp, frame, frame_index, ip)
            n, m, dt = check_meta(rec, f"Integrate() of frame {frame_index}")
            checked += n
            merges, detached = max(merges, m), max(detached, dt)
            # two sweeps at the same frame with different windows: each makes the other buffer current
            for w in (window, window + 2):
                rec.Regularize(None, frame_index, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, w)
                n, _, _ = check_meta(rec, f"Regularize() of frame {frame_index}, window {w}")
                checked += n
        assert checked > 0
        assert merges > 0, "the sequence should include merges"
        assert detached > 0, "the sequence should include surfels with the detach flag"
    finally:
        rec.close()
