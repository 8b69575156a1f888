"""Every frame the frame loop integrates through its other input paths, held to the walks (tests/frame_loop_walk.py)
push by push, as tests/test_frame_loop_walk_gpu.py holds the frames pushed at the handle's size with known poses:

  --pyramid_level L     full-size frames downscaled into the ring (StageDownscaleMedian, StageColorPyramid), device
                        frames read in place and host frames through the full-size staging; L = 3 downscales in the
                        warp-per-pixel kernel;
  median densify n      the MedianFilterAndDensifyDepthMap passes through median_stage[0] (and median_stage[1] from
                        n = 2 on) into the ring;
  mixed pushes          one session whose pushes rotate device -> pageable -> pinned frames, so consecutive uploads
                        alternate between the work stream and the upload stream over the shared staging;
  pose-free sessions    TrackedSession (depth only, with colour, with relocalisation): the poses come from the tracker,
                        which renders the cloud between pushes while frames are in flight. With relocalisation a lost
                        frame is left out, and the chain's frame index counts pushes, not source frames.

Each frame's inputs are the raw frames after the stage hook of the path (FW.stage_pyramid, FW.stage_median),
pre-processed on a second handle with the outlier-filter transforms of the pushed poses. The streams are
test_frame_loop_walk_gpu.make_stream's: their first frames see the scene nearer, which reaches the conflicting-surfel
and replacement branches.

Not held: the frames sm_session_end integrates in the frame-graph mode. It runs its last two steps without returning
to the caller, so they cannot be dumped one by one.
"""
import functools
import time

import pytest
import torch

from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200 import synthetic as S
from surfelmeshing_b200._lib import RelocParams, TrackRGBDParams
from tests import frame_loop_walk as FW
from tests import reloc_walk as RW
from tests.test_frame_loop_walk_gpu import CAP, FRAMES, QVGA, VGA, make_stream, params, session_chain, stream_run_chain

pytestmark = pytest.mark.gpu

KINDS = ("device", "pageable", "pinned")


@functools.lru_cache(maxsize=None)
def full_stream(width, height, frames=FRAMES):
    """make_stream at a sensor size 2^L times the handle's (shared by the chains of one size; none writes to it)."""
    return make_stream(S.Camera.tum(width, height), frames)


def pyramid_chain(label, level, full_size, kinds, **kw):
    full = S.Camera.tum(*full_size)
    cam = full.scaled(level)
    return session_chain(label, cam=cam, st=full_stream(*full_size), kinds=kinds,
                         stage=FW.stage_pyramid(level, cam.width, cam.height), configure=(("pyramid_level", level),),
                         **kw)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("level,full_size", [(1, (640, 480)), (2, (1280, 960))], ids=["L1", "L2"])
def test_pyramid_session_chain(product, level, full_size, kind):
    """A 320 x 240 handle fed 2^L times larger frames."""
    pyramid_chain(f"pyramid L{level} {kind}", level, full_size, (kind,))


def test_pyramid_level_3_session_chain(product):
    """A 160 x 120 handle fed 1280 x 960 frames: 8 x 8 blocks, the warp-per-pixel downscale kernel."""
    pyramid_chain("pyramid L3 device", 3, (1280, 960), ("device",))


@pytest.mark.parametrize("passes", [1, 3])
def test_median_densify_session_chain(product, passes):
    """n = 1 writes the one pass straight into the ring slot; n = 3 ping-pongs through median_stage[1]."""
    session_chain(f"median densify n={passes}", stage=FW.stage_median(passes),
                  configure=(("median_filter_and_densify_iterations", passes),))


def test_pyramid_session_with_mixed_pushes(product):
    """Pushes rotate device -> pageable -> pinned frames: a device frame is downscaled in place on the work stream, a
    host frame staged full-size and downscaled on the upload stream, into consecutive ring slots."""
    pyramid_chain("pyramid L1 mixed pushes", 1, (640, 480), KINDS)


def test_median_densify_session_with_mixed_pushes(product):
    """As above with two median passes: both streams write median_stage[0] and median_stage[1] in turn."""
    session_chain("median densify n=2 mixed pushes", kinds=KINDS, stage=FW.stage_median(2),
                  configure=(("median_filter_and_densify_iterations", 2),))


def test_pyramid_stream_run_one_frame_per_call(product):
    """sm_stream_run over [f, f + 1) at L = 1 with the full-size frames in pinned memory: each call stages its frames
    full-size on the upload stream before the downscale."""
    full = S.Camera.tum(640, 480)
    cam = full.scaled(1)
    stream_run_chain("stream_run [f, f + 1) pyramid L1 pinned", cam=cam, st=full_stream(640, 480, 24),
                     frames_on=lambda a: a.cpu().pin_memory(), stage=FW.stage_pyramid(1, cam.width, cam.height),
                     configure=(("pyramid_level", 1),))


# ---------------------------------------------------------------------------------------------
# pose-free sessions
# ---------------------------------------------------------------------------------------------

def tracked_chain(label, cam, depth, color, first_pose, frames, rgbd=None, reloc=None, hold_from=0, min_frames=15,
                  waive=()):
    """A TrackedSession holding every frame it integrates from frame index `hold_from` on, with the poses it pushed.
    depth / color: the source frames (CUDA tensors, pushed in place). Returns the session."""
    pp, ip = params(cam)
    rec = R.CUDASurfelReconstruction(CAP, *FW.camera_tuple(cam))
    sources, global_T, frame_T = [], [], []
    chain = FW.Chain(label, rec, FW.Inputs(cam, depth, color, pp, sources=sources), ip, (global_T, frame_T))
    t0 = time.perf_counter()
    last = -1
    try:
        with R.TrackedSession(rec, pp, ip, first_pose, rgbd=rgbd, reloc=reloc) as s:
            for f in range(frames):
                status = s.push(depth[f], color[f])
                if status is None:
                    continue
                pose = s.trajectory[f]
                sources.append(f)
                global_T.append(pose)
                frame_T.append(R.invert_rigid(pose))
                g = status.last_integrated_frame
                if g != last:
                    assert last < 0 or g == last + 1, f"{label}: source frame {f} integrated up to {g} after {last}"
                    if g >= hold_from:
                        chain.hold(g)
                    elif g == hold_from - 1:
                        chain.restart()
                    last = g
        chain.finish(min_frames, waive)
    finally:
        rec.close()
    assert sources == FW.pushed_sources(s.states, held_out=reloc is not None)
    print(f"{label}: {time.perf_counter() - t0:.1f} s")
    return s


@pytest.mark.parametrize("rgbd", [False, True], ids=["depth", "rgbd"])
def test_tracked_session_chain(product, rgbd):
    """The QVGA stream tracked from frame 0's pose alone. The tracker meets the change of scale after the nearer
    frames like a sensor whose depth scale drifts: whatever it tracks is the pose pushed, and the pose held."""
    st = make_stream(QVGA, FRAMES)
    tracked_chain(f"tracked {'rgbd' if rgbd else 'depth'}", QVGA, st.depth, st.color, st.global_T_frame[0], FRAMES,
                  rgbd=TrackRGBDParams.defaults() if rgbd else None)


MAPPED = 150     # test_reloc_gpu.py::test_pose_free_session_relocalises_after_a_jump
HOLD_FROM = 140


def test_tracked_session_chain_relocalises_after_a_jump(product):
    """test_reloc_gpu's jump stream: 150 VGA frames, an empty frame, then a jump back to orbit frames 60-79. The chain
    holds the frames from push 140 on (before it, only the state after push 139's frame is taken), across the lost
    frame left out and the relocalised one. The stream is test_reloc_gpu's, without nearer frames: its static scene reaches no
    conflicting surfel and no replacement (0 of each over the 24 frames held), so this chain waives those two floors;
    the other chains here reach them, and what this one adds is the frames left out and the relocalised pose."""
    st = S.make_stream(VGA, MAPPED, device="cuda")
    tail = RW.jump_frames(VGA, 60, 20)
    # a sensor dropout (no valid depth) between the mapped frames and the jump: tracking loses it and relocalisation
    # has nothing to match, so it is left out (the jump's first frame relocalises at once)
    depth = list(st.depth) + [torch.zeros_like(st.depth[0])] + [d for d, _, _ in tail]
    color = list(st.color) + [st.color[-1]] + [c for _, c, _ in tail]
    s = tracked_chain("tracked reloc jump", VGA, depth, color, st.global_T_frame[0], len(depth),
                      reloc=RelocParams.defaults(), hold_from=HOLD_FROM, min_frames=12,
                      waive=("replacements", "conflicting surfels"))
    assert "relocalised" in s.states[MAPPED:] and "lost" in s.states[MAPPED:], s.states[MAPPED:]
