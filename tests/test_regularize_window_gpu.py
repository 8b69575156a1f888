"""Regularize() keeps the smooth position of every slot outside the regularisation window bit for bit.

k_reg_step rewrites only the slots that are in the window or were in it at the previous sweep; every other
writer of smooth positions (merges, replacements, new surfels, Integrate() without denoising) keeps both
smooth buffers equal for the slots it touches. A slot that was skipped although its two buffers differ shows
up here as a changed out-of-window smooth position."""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams
from tests.util import SMOOTH_ROWS, other_frames

pytestmark = pytest.mark.gpu

STAMP_ROW = R.ROW_NAMES.index("last_update_stamp")
W, H = 320, 240


@pytest.fixture(scope="module")
def stream():
    cam = S.Camera.tum(W, H)
    st = S.make_stream(cam, 40, stream_id=3, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    torch.cuda.synchronize()
    return cam, st, pp


def integrate(rec, st, pp, frame, frame_index, ip):
    others = [st.depth[f] for f in other_frames(frame, pp.outlier_filtering_frame_count)]
    d = torch.zeros((H, W), dtype=torch.uint16, device="cuda")
    n = torch.zeros((H, W, 2), device="cuda")
    r = torch.zeros((H, W), device="cuda")
    rec.preprocess(None, pp, st.depth[frame], others, st.others_TR_reference[frame], d, n, r)
    rec.integrate(None, frame_index, ip, d, n, r, st.color[frame], st.global_T_frame[frame], st.frame_T_global[frame])


def regularize_and_check(rec, frame_index, window, ip):
    before, n, _ = rec.dump_state()
    rec.Regularize(None, frame_index, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors, window)
    after, n_after, _ = rec.dump_state()
    assert n_after == n
    stamps = before[STAMP_ROW].view(np.uint32).astype(np.int64)
    threshold = np.int32(np.uint32(frame_index) - np.uint32(window)).item()
    outside = stamps < threshold
    smooth_before = before[list(SMOOTH_ROWS)][:, outside].view(np.uint32)
    smooth_after = after[list(SMOOTH_ROWS)][:, outside].view(np.uint32)
    changed = int((smooth_before != smooth_after).any(axis=0).sum())
    assert changed == 0, f"{changed} of {int(outside.sum())} out-of-window slots moved (frame {frame_index}, window {window})"
    return int(outside.sum()), n


# (stream frame, frame index, regularization_frame_window_size, regularisation iterations inside Integrate(),
#  action before the step)
SEQUENCES = {
    "skips_and_windows": [(f, 3 * f, w, 1, None) for f, w in zip(range(4, 30), [2, 5, 3, 8, 2, 1, 4] * 4)],
    "denoising_off_between": [(f, 2 * f, 3, 0 if f % 3 == 1 else 1, None) for f in range(4, 30)],
    "load_state_and_reset": (
        [(f, 2 * f, 4, 1, None) for f in range(4, 14)]
        + [(14, 28, 4, 1, "reload")]
        + [(f, 2 * f, 6, 1, None) for f in range(15, 22)]
        + [(22, 5, 3, 1, "reset")]  # frame indices start over below the previous threshold
        + [(f, f - 17, 3, 2, None) for f in range(23, 34)]
    ),
}


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_out_of_window_smooth_positions_stay(product, stream, name):
    cam, st, pp = stream
    rec = R.CUDASurfelReconstruction(400_000, W, H, cam.fx, cam.fy, cam.cx, cam.cy)
    checked = merges = 0
    try:
        for frame, frame_index, window, iterations, action in SEQUENCES[name]:
            if action == "reload":
                rows, _, merge_count = rec.dump_state()
                rec.load_state(rows, merge_count)
            elif action == "reset":
                rec.reset()
            ip = IntegrateParams.defaults()
            ip.regularization_frame_window_size = window
            ip.regularization_iterations_per_integration_iteration = iterations
            integrate(rec, st, pp, frame, frame_index, ip)
            merges = max(merges, rec.dump_state()[2])
            outside, _ = regularize_and_check(rec, frame_index, window, ip)
            checked += outside
            # a second sweep at the same frame with another window
            outside, _ = regularize_and_check(rec, frame_index, window + 2, ip)
            checked += outside
        assert checked > 0
        assert merges > 0, "the sequence should include merges"
    finally:
        rec.close()
