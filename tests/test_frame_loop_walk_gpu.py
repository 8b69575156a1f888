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
pre-processing to that call, so a difference here is a finding about the pre slot of the graph.

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
from tests.util import other_frames

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


def camera_tuple(cam):
    return cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy


class Inputs:
    """The pre-processed inputs of a stream's frames, from a handle of their own."""

    def __init__(self, cam, st, pp):
        self.cam, self.st, self.pp = cam, st, pp
        self.rec = R.CUDASurfelReconstruction(1024, *camera_tuple(cam))

    def frame(self, local):
        cam, st, pp = self.cam, self.st, self.pp
        K = pp.outlier_filtering_frame_count
        others = [st.depth[f] for f in other_frames(local, K)]
        transforms = R.outlier_filter_transforms(st.global_T_frame, st.frame_T_global, local, K, pp.depth_scaling)
        H, W = cam.height, cam.width
        d = torch.zeros((H, W), dtype=torch.uint16, device="cuda")
        n = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
        r = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        self.rec.preprocess(None, pp, st.depth[local], others, transforms, d, n, r)
        torch.cuda.synchronize()
        return dict(depth_pre=d.cpu().numpy(), normals=n.cpu().numpy(), radius=r.cpu().numpy(),
                    color=st.color[local].cpu().numpy())

    def close(self):
        self.rec.close()


class Chain:
    """Holds frame after frame of one handle, each from the state the previous hold (or a call between) left."""

    def __init__(self, label, rec, cam, st, pp, ip, first_frame_index=0, plain=False):
        self.label, self.rec, self.cam, self.st, self.ip = label, rec, cam, st, ip
        self.first = first_frame_index
        self.winner = "plain" if plain else "member"
        self.inputs = Inputs(cam, st, pp)
        self.rows, self.merges = np.zeros((25, 0), np.float32), 0
        self.totals = FW.Totals(label)

    def restart(self):
        """The state after a call between pushes: the next frame starts from it."""
        rows, _, merges = self.rec.dump_state()
        self.rows, self.merges = rows.copy(), merges

    def hold(self, frame_index):
        rec, st = self.rec, self.st
        local = frame_index - self.first
        rows, n, merges = rec.dump_state()
        rows = rows.copy()
        rasters = rec.download_rasters()
        counters = FW.frame_counters(rec)
        stats = FW.hold_frame(self.rows, rows, merges, rasters, self.inputs.frame(local), frame_index,
                              st.global_T_frame[local], st.frame_T_global[local], camera_tuple(self.cam), self.ip,
                              merges_before=self.merges, counters=counters, winner=self.winner,
                              label=f"{self.label} frame {frame_index}")
        self.totals.add(stats)
        self.rows, self.merges = rows, merges

    def finish(self, min_frames):
        self.inputs.close()
        print(self.totals.report())
        self.totals.assert_floors(min_frames)


def params(cam, K=8):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    pp.outlier_filtering_frame_count = K
    return pp, IntegrateParams.defaults()


def session_chain(label, cam=QVGA, frames=FRAMES, K=8, pp_set=None, ip_set=None, plain=False, serial=False,
                  first_frame_index=0, pinned=False, between=None, min_frames=15):
    pp, ip = params(cam, K)
    for k, v in (pp_set or {}).items():
        setattr(pp, k, v)
    for k, v in (ip_set or {}).items():
        setattr(ip, k, v)
    st = make_stream(cam, frames, K)
    rec = R.CUDASurfelReconstruction(CAP, *camera_tuple(cam))
    if plain:
        rec.configure("tiebreak_wave", 0)
    if serial:
        rec.enable_timings(True)
    chain = Chain(label, rec, cam, st, pp, ip, first_frame_index, plain)
    t0 = time.perf_counter()
    last = -1
    try:
        with rec.session(pp, ip, (cam.width, cam.height), first_frame_index) as s:
            for i in range(frames):
                d, c = st.depth[i], st.color[i]
                if pinned:
                    d, c = d.cpu().pin_memory(), c.cpu().pin_memory()
                status = s.push(d, c, st.global_T_frame[i], st.frame_T_global[i])
                f = status.last_integrated_frame
                if f != last:
                    assert last < 0 or f == last + 1, f"{label}: push {i} integrated up to {f} after {last}"
                    chain.hold(f)
                    last = f
                    if between is not None and between(s, rec, f, ip):
                        chain.restart()
        chain.finish(min_frames)
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
    "pinned-host-frames": dict(pinned=True),
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


def test_stream_run_one_frame_per_call(product):
    """sm_stream_run over [f, f + 1), sixteen times on one handle: every call runs the graph's placeholder steps around
    its one frame, and continues from the state the previous call left."""
    cam = QVGA
    pp, ip = params(cam)
    st = make_stream(cam, 24)
    others = R.stream_outlier_filter_transforms(st.global_T_frame, st.frame_T_global, 8, st.depth_scaling)
    rec = R.CUDASurfelReconstruction(CAP, *camera_tuple(cam))
    chain = Chain("stream_run [f, f + 1)", rec, cam, st, pp, ip)
    try:
        for f in range(4, 20):
            stats = rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, others, pp, ip, f, f + 1)
            assert stats.frames_integrated == 1
            chain.hold(f)
        chain.finish(min_frames=16)
    finally:
        rec.close()
