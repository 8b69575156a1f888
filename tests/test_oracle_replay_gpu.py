"""Oracle replay of a free-running product: teacher forcing the other way round.

The product runs a stream uninterrupted and never reloads its state, so its regularisation keeps the state it
carries between sweeps (the two smooth record buffers and the previous sweep's window threshold, which lets
k_reg_step skip the slots that were already outside the window then). Before every step the product's dumped state
is loaded into the oracle handles (A, and the B runs that measure the reference's own envelope), and all run the step on the product's pre-processed inputs. The
reference keeps no state outside the surfel rows (it clears its gradient rows at the start of every sweep), so any
difference in what the step leaves comes from the product's hidden state or its kernels.
"""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams
from tests.test_parity_gpu import ORACLE_B_RUNS, compare_integrate, compare_smooth, frame_walk, u16
from tests.util import INTEGRATE_ROWS, NEIGHBOR_ROWS, count_mismatch, other_frames, regularization_threshold

pytestmark = pytest.mark.gpu

CAM = S.Camera.tum(320, 240)
FRAMES = 24      # 16 integrated frames
FRAME_STEP = 3   # frame index = 3 x stream frame: slots leave the 30-frame default window within the stream
CAP = 400_000

# Regularize() settings of the standalone sequence, one after the other: (window, weight, radius factor)
REGULARIZE_SETTINGS = [(2, 2.0, 1.5), (5, 10.0, 2.0), (30, 40.0, 3.0), (2, 40.0, 2.0), (30, 2.0, 3.0), (5, 40.0, 1.5),
                       (30, 10.0, 1.5), (2, 10.0, 3.0), (5, 2.0, 2.0)]

SEQUENCES = {
    "defaults": {},
    "window3": {"regularization_frame_window_size": 3},
    "reg2": {"regularization_iterations_per_integration_iteration": 2},
    "denoise_off_every_third": {},
    "standalone_regularize": {},
}


def make(lib=None):
    return R.CUDASurfelReconstruction(CAP, CAM.width, CAM.height, CAM.fx, CAM.fy, CAM.cx, CAM.cy, lib=lib)


def left_the_window(rows, previous_threshold, threshold):
    """Live slots that were inside the window of the previous k_reg_step sweep and are outside this one's: the
    slots the partial sweep must carry over from one record buffer to the other."""
    if previous_threshold is None:
        return 0
    stamps = rows[18].view(np.int32)
    return int(((stamps >= previous_threshold) & (stamps < threshold) & (rows[7] >= 0)).sum())


def reload(rec_p, oracles):
    rows, n, merges = rec_p.dump_state()
    for rec in oracles:
        rec.load_state(rows, merges)
    return rows, n


def compare_regularize(rec_p, rec_a, recs_b, frame_index, window, n):
    """Regularize() on one state: smooth positions as compare_smooth; every other row the call reads or writes,
    the neighbour links included (far-neighbour pruning), bit-exact."""
    (rows_p, n_p, m_p), (rows_a, n_a, m_a) = rec_p.dump_state(), rec_a.dump_state()
    assert (n_p, m_p) == (n_a, m_a)
    for row in INTEGRATE_ROWS + NEIGHBOR_ROWS:
        assert count_mismatch(rows_p[row], rows_a[row]) == 0, f"row {row}"
    compare_smooth(rows_p, rows_a, frame_index, window, 1, rows_b=[rec.dump_state()[0] for rec in recs_b], n_before=n,
                   label=f"Regularize({frame_index}, window {window}): ")


@pytest.mark.parametrize("sequence", list(SEQUENCES))
def test_replay_free_running_product(product, reference, sequence):
    st = S.make_stream(CAM, FRAMES, stream_id=21, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = CAM.valid_region_radius()
    ip = IntegrateParams.defaults()
    for k, v in SEQUENCES[sequence].items():
        setattr(ip, k, v)
    rec_p, rec_a = make(), make(reference)
    recs_b = [make(reference) for _ in range(ORACLE_B_RUNS)]
    W, H = CAM.width, CAM.height
    first, last = st.integrated_range()
    previous_threshold = None   # int(frame - window) of the product's previous k_reg_step sweep
    partial_steps = 0
    for step, frame in enumerate(range(first, last)):
        index = FRAME_STEP * frame
        ipf = IntegrateParams.from_buffer_copy(ip)
        if sequence == "denoise_off_every_third" and step % 3 == 2:
            ipf.regularization_iterations_per_integration_iteration = 0
        others = [st.depth[f] for f in other_frames(frame, pp.outlier_filtering_frame_count)]
        d0, n0, r0 = u16(H, W), torch.zeros((H, W, 2), device="cuda"), torch.zeros((H, W), device="cuda")
        rec_p.preprocess(None, pp, st.depth[frame], others, st.others_TR_reference[frame], d0, n0, r0)
        rows, n_before = reload(rec_p, [rec_a] + recs_b)
        dp, da = d0.clone(), d0.clone()
        for rec, d in [(rec_p, dp), (rec_a, da)] + [(rec_b, d0.clone()) for rec_b in recs_b]:
            rec.integrate(None, index, ipf, d, n0, r0, st.color[frame], st.global_T_frame[frame], st.frame_T_global[frame])
        torch.cuda.synchronize()
        state_p = rec_p.dump_state()
        compare_integrate(rec_p.download_rasters(), dp.cpu().numpy(), state_p, rec_a.download_rasters(),
                          da.cpu().numpy(), rec_a.dump_state(), n_before,
                          states_b=[rec.dump_state() for rec in recs_b], ip=ipf, frame_index=index,
                          walk=frame_walk(rows, index, CAM, st, d0, n0, ipf, stream_frame=frame))
        if ipf.regularization_iterations_per_integration_iteration > 0:
            threshold = regularization_threshold(index, ipf.regularization_frame_window_size)
            partial_steps += left_the_window(state_p[0], previous_threshold, threshold) > 0
            previous_threshold = threshold
        if sequence == "standalone_regularize":
            window, weight, radius_factor = REGULARIZE_SETTINGS[step % len(REGULARIZE_SETTINGS)]
            rows, n = reload(rec_p, [rec_a] + recs_b)
            for rec in [rec_p, rec_a] + recs_b:
                rec.Regularize(None, index, weight, radius_factor, window)
            torch.cuda.synchronize()
            threshold = regularization_threshold(index, window)
            partial_steps += left_the_window(rows, previous_threshold, threshold) > 0
            previous_threshold = threshold
            compare_regularize(rec_p, rec_a, recs_b, index, window, n)
    print(f"{sequence}: {partial_steps} sweeps with slots that left the window since the previous sweep")
    assert partial_steps > 0, "the partial sweep never had slots to carry over"
