"""Every frame the frame loop integrates, held to the walks (tests/frame_loop_walk.py) from the loop's own previous
state, push by push.

The frame graph runs each frame in three steps (crit: integrate, scan, update_neighbors, create and the
regularisation sweeps of frame f; front: project, associate, merge and blend of frame f + 1; pre: the pre-processing
and raster clears of frame f + 2), rotates three buffer sets, two smooth buffers and the count slots between steps,
and is ordered by nothing but the graph's edges. A session hands the state back between pushes: after every push that
integrates a frame, the chain dumps the state and the rasters, and holds that frame to the walk of the state it
started from (the previous dump, or the dump after a call between the pushes). A missing edge, a front half that
reads a buffer one rotation early, a smooth buffer not carried into the next step, a ring slot reused too soon or a
stale raster after a compaction re-runs the front half fails the first frame it touches, where the surfel counts of a
whole stream would only drift.

Each frame's inputs come from a second handle outside the session: `preprocess` of the raw frame with the
outlier-filter transforms of the pushed poses. The first-frame parity tests hold the frame loop's fused
pre-processing to that call, so a difference here is a finding about the pre slot of the graph. The chains here push
raw frames at the handle's size with the stream's poses; tests/test_frame_loop_inputs_gpu.py holds the pyramid,
median-densify and pose-free paths with the same Chain.

Not held: the frames sm_session_end integrates in the frame-graph mode. It runs its last two steps without returning
to the caller, so they cannot be dumped one by one.
"""
import time

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200 import synthetic as S
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams
from tests import frame_loop_walk as FW
from tests.test_reloc_gpu import odd_camera

pytestmark = pytest.mark.gpu

QVGA = S.Camera.tum(320, 240)
VGA = S.Camera.tum(640, 480)
CAP = 2_000_000
FRAMES = 28


NEARER_UNTIL = 10     # the frames before this one see the scene 15 % nearer


def make_stream(cam, frames, K=8):
    """The synthetic stream with its first frames' depths scaled by 0.85: a surface that later moves away (or a sensor
    whose depth scale drifts). The frames from NEARER_UNTIL on meet the surfels the early frames left in front of their
    measurements, which reaches the conflicting-surfel, confidence-decrement and replacement branches of the cycle; a
    static scene never does (0 of each over every chain here without it). The outlier filter keeps the scaled frames,
    which agree with each other to well within its tolerance at these camera speeds."""
    st = S.make_stream(cam, frames, stream_id=41, device="cuda", other_count=K)
    near = st.depth[:NEARER_UNTIL].to(torch.int32)
    st.depth[:NEARER_UNTIL] = ((near * 17 + 10) // 20).to(torch.uint16)
    return st


camera_tuple = FW.camera_tuple


def params(cam, K=8):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    pp.outlier_filtering_frame_count = K
    return pp, IntegrateParams.defaults()


def host_frame(a, kind):
    """A frame tensor as pushed: "device" (CUDA, read in place), "pageable" or "pinned" host memory."""
    return a if kind == "device" else (a.cpu().pin_memory() if kind == "pinned" else a.cpu())


def session_chain(label, cam=QVGA, frames=FRAMES, K=8, pp_set=None, ip_set=None, plain=False, serial=False,
                  first_frame_index=0, kinds=("device",), between=None, min_frames=15, st=None,
                  stage=FW.stage_identity, configure=(), waive=()):
    """A session on a handle at `cam` holding every frame it integrates. st: the stream (default: make_stream at cam),
    its frames pushed as they are (at 2^L x cam with configure pyramid_level L) and held after `stage`; push i gives
    kinds[i % len(kinds)] frames; configure: sm_configure (key, value) pairs."""
    pp, ip = params(cam, K)
    for k, v in (pp_set or {}).items():
        setattr(pp, k, v)
    for k, v in (ip_set or {}).items():
        setattr(ip, k, v)
    st = st or make_stream(cam, frames, K)
    rec = R.CUDASurfelReconstruction(CAP, *camera_tuple(cam))
    if plain:
        rec.configure("tiebreak_wave", 0)
    if serial:
        rec.enable_timings(True)
    for key, value in configure:
        rec.configure(key, value)
    chain = FW.Chain(label, rec, FW.Inputs(cam, st.depth, st.color, pp, stage), ip,
                     (st.global_T_frame, st.frame_T_global), first_frame_index, plain)
    t0 = time.perf_counter()
    last = -1
    try:
        with rec.session(pp, ip, (st.depth.shape[2], st.depth.shape[1]), first_frame_index) as s:
            for i in range(frames):
                kind = kinds[i % len(kinds)]
                d, c = host_frame(st.depth[i], kind), host_frame(st.color[i], kind)
                status = s.push(d, c, st.global_T_frame[i], st.frame_T_global[i])
                f = status.last_integrated_frame
                if f != last:
                    assert last < 0 or f == last + 1, f"{label}: push {i} integrated up to {f} after {last}"
                    chain.hold(f)
                    last = f
                    if between is not None and between(s, rec, f, ip):
                        chain.restart()
        chain.finish(min_frames, waive)
    finally:
        rec.close()
    print(f"{label}: {time.perf_counter() - t0:.1f} s")
    return chain.totals


CASES = {
    "defaults": dict(),
    "no-regularisation": dict(ip_set=dict(regularization_iterations_per_integration_iteration=0,
                                          regularization_frame_window_size=-1)),
    "no-blending": dict(ip_set=dict(do_blending=0)),
    "plain-tiebreak": dict(plain=True),
    "odd-camera-K4": dict(cam=odd_camera(), K=4),
    "bilateral-radius-4": dict(pp_set=dict(bilateral_filter_sigma_xy=2.0)),
    "first-frame-2^30-64": dict(first_frame_index=2**30 - 64),
    "pinned-host-frames": dict(kinds=("pinned",)),
    "serial": dict(serial=True),
}


def test_session_chain_with_calls_between_pushes(product):
    """sm_compact after two pushes (the session re-runs the front half of the frame in flight on the compacted state,
    and the merge count restarts at 0) and sm_regularize after two others: the next frame starts from the state the
    call left."""
    done = []

    def between(s, rec, f, ip):
        if f in (9, 17):
            stats = s.compact()
            assert stats.slots_after < stats.slots_before and rec.dump_state()[2] == 0
        elif f in (12, 20):
            rec.Regularize(None, f, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors,
                           ip.regularization_frame_window_size)
        else:
            return False
        done.append(f)
        return True

    session_chain("calls-between-pushes", between=between)
    assert done == [9, 12, 17, 20]


@pytest.mark.parametrize("case", list(CASES))
def test_session_chain(product, case):
    totals = session_chain(case, **CASES[case])
    if case == "no-blending":   # the walk is fed the pre-processed depth itself: nothing is ranged or excused
        assert totals.ranged == 0 and totals.excused == 0 and totals.excused_frames == 0


def test_session_chain_vga(product):
    session_chain("640x480", cam=VGA, frames=24, min_frames=12)


def stream_run_chain(label, cam=QVGA, st=None, frames_on=lambda a: a, stage=FW.stage_identity, configure=()):
    """sm_stream_run over [f, f + 1), sixteen times on one handle, holding each frame. st: the stream (default:
    make_stream at cam), passed through frames_on (e.g. into pinned memory) and held after `stage`."""
    pp, ip = params(cam)
    st = st or make_stream(cam, 24)
    others = R.stream_outlier_filter_transforms(st.global_T_frame, st.frame_T_global, 8, st.depth_scaling)
    rec = R.CUDASurfelReconstruction(CAP, *camera_tuple(cam))
    for key, value in configure:
        rec.configure(key, value)
    chain = FW.Chain(label, rec, FW.Inputs(cam, st.depth, st.color, pp, stage), ip,
                     (st.global_T_frame, st.frame_T_global))
    depth, color = frames_on(st.depth), frames_on(st.color)
    t0 = time.perf_counter()
    try:
        for f in range(4, 20):
            stats = rec.stream_run(None, depth, color, st.global_T_frame, st.frame_T_global, others, pp, ip, f, f + 1)
            assert stats.frames_integrated == 1
            chain.hold(f)
        chain.finish(min_frames=16)
    finally:
        rec.close()
    print(f"{label}: {time.perf_counter() - t0:.1f} s")


def test_stream_run_one_frame_per_call(product):
    """sm_stream_run over [f, f + 1), sixteen times on one handle: every call runs the graph's placeholder steps around
    its one frame, and continues from the state the previous call left."""
    stream_run_chain("stream_run [f, f + 1)")
