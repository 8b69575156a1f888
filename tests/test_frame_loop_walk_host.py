"""The per-frame hold of tests/frame_loop_walk.py on the recorded reference frames, and its frame-excuse rule on a
constructed frame. CPU only: this is where the composition of the walks is checked without a GPU."""
import numpy as np
import pytest

from tests import frame_loop_walk as FW
from tests import integrate_walk as IW
from tests.test_integrate_walk_host import integrate_params
from tests.util import golden_camera, golden_params, load_golden


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def golden_frame(g, f):
    return dict(depth_pre=g[f"f{f}_pre_depth"], normals=g[f"f{f}_normals"], radius=g[f"f{f}_radius"], color=g["color"][f])


def test_recorded_frames_5_to_7(golden):
    """Frames 5-7 of the recording, each from the recorded state before it: association, the blend from the recorded
    counts and sums, the cycle, the smooth positions against the regularisation sweep the recording ran (defaults:
    one sweep, window 30) and the merge count. The reference applies a merge in place, so the slots whose merge
    partner merges in the same frame are excused."""
    ip = golden_params(golden)[1]
    assert ip.regularization_iterations_per_integration_iteration == 1 and ip.do_blending
    totals = FW.Totals("golden frames 5-7")
    for f in (5, 6, 7):
        rasters = {k[len(f"f{f}_"):]: v for k, v in golden.items() if k.startswith(f"f{f}_")}
        n_after, merges = [int(v) for v in golden[f"f{f}_counts"]]
        stats = FW.hold_frame(golden[f"f{f - 1}_state"], golden[f"f{f}_state"], merges, rasters, golden_frame(golden, f),
                              f, golden["global_T_frame"][f], golden["frame_T_global"][f], golden_camera(golden), ip,
                              merges_before=int(golden[f"f{f - 1}_counts"][1]), merge_chains_excused=True,
                              label=f"golden frame {f}")
        assert n_after == stats["slots"]
        assert "reg_close" in stats
        print(f"golden frame {f}: {stats}")
        totals.add(stats)
    print(totals.report())
    totals.assert_fractions()
    assert totals.floors()["merges"] > 0 and totals.floors()["integrations"] > 0 and totals.new > 0


# A 16 x 12 frame: supported surfels on the left half at 1 m, 0.2 mm in front of the measurement; on the right half
# unsupported measurements at 1 m, and one pixel U measured at 1 unit (0.2 mm). U lies on the surfel-border ring of
# the blend: its blended depth is 1.5 + (surfel - measurement) x 2500 units at radius 3, which lands on 1.0 up to the
# reciprocal of the depth scaling, so its range is [0, 1]: created with the upper end, not with the lower.
SMALL = (16, 12, 14.0, 14.0, 8.0, 6.0)
U = (6, 8)   # (y, x)


def constructed_frame(u_depth):
    W, H, fx, fy, cx, cy = SMALL
    ip = integrate_params(2**31 - 1, 1)
    ip.measurement_blending_radius = 3
    ip.regularization_iterations_per_integration_iteration = 0
    depth = np.full((H, W), 5000, np.uint16)
    depth[U] = u_depth
    supported = np.zeros((H, W), bool)
    supported[:, :8] = True
    z_surfel = np.float32(1.0 - 0.0002)
    ys, xs = np.nonzero(supported)
    n = len(ys)
    rows = np.zeros((IW.ROW_COUNT, n), np.float32)
    rows[0] = (xs + 0.5 - cx) / fx * z_surfel
    rows[1] = (ys + 0.5 - cy) / fy * z_surfel
    rows[2] = z_surfel
    rows[3:6] = rows[0:3]
    rows[6] = 1.0
    rows[7] = (1.2 / fx) ** 2
    rows[10] = -1.0
    ru = rows.view(np.uint32)
    ru[17] = ru[18] = 3
    ru[19:23] = IW.INVALID
    ru[24] = 0x808080
    supporting = np.full((H, W), IW.INVALID, np.uint32)
    supporting[ys, xs] = np.arange(n, dtype=np.uint32)
    rasters = dict(supporting_surfels=supporting, supporting_surfel_counts=supported.astype(np.uint32),
                   supporting_surfel_depth_sums=np.where(supported, z_surfel, np.float32(0)).astype(np.float32),
                   conflicting_surfels=np.full((H, W), IW.INVALID, np.uint32),
                   first_surfel_depth=np.where(supported, z_surfel, np.float32(np.inf)).astype(np.float32))
    frame = dict(depth_pre=depth, normals=np.zeros((H, W, 2), np.float32),
                 radius=np.full((H, W), (1.2 / fx) ** 2, np.float32), color=np.full((H, W, 3), 100, np.uint8))
    return rows, rasters, frame, ip


def test_a_ranged_pixel_that_flips_a_creation_excuses_the_frame(monkeypatch):
    """With U measured at 1 unit, the blend leaves U in [0, 1]: whether a surfel is created there is open, and with it
    the index of every later new surfel, so the frame is excused whatever the run's rows are. Measured at 2 units,
    U is created either way: the frame is compared, and U's new surfel, whose position is the ranged depth's, is one
    of the excused slots."""
    eye = np.eye(4, dtype=np.float32)[:3]
    for u_depth, flips in ((1, True), (2, False)):
        rows, rasters, frame, ip = constructed_frame(u_depth)
        bl = IW.blend(frame["depth_pre"], rasters["supporting_surfel_counts"], rasters["supporting_surfel_depth_sums"],
                      3, ip.depth_scaling)
        assert (int(bl.lo[U]), int(bl.hi[U])) == ((0, 1) if flips else (1, 2)), (bl.lo[U], bl.hi[U])
        res = IW.walk(rows, dict(frame, depth=bl.depth), rasters, SMALL, ip, 4, eye, eye)
        out = {k: v for k, v in rasters.items()}
        out.update(new_surfel_flag_vector=res.new_flag, new_surfel_indices=res.new_index)
        # the association of the constructed state is not the point here: the rasters are taken as the run's
        monkeypatch.setattr(IW, "hold_association", lambda *a, **k: {})
        stats = FW.hold_frame(rows, res.rows, 0, out, frame, 4, eye, eye, SMALL, ip, label=f"U at {u_depth}")
        print(f"U measured at {u_depth}: {stats}")
        assert stats["excused_frame"] == int(flips)
        if not flips:
            assert res.new_flag[U] == 1
            assert stats["excused"] >= 1 and stats["ranged"] >= 1


# ---------------------------------------------------------------------------------------------
# the inputs of a chain: stage hooks and the push -> source frame map
# ---------------------------------------------------------------------------------------------

def test_stage_hooks_on_recorded_frames(golden):
    """Inputs' staged frames are the pyramid / median restatements of each recorded frame alone, whatever order the
    frames are staged in and however often each is read (a frame is read as its neighbours' outlier frame too)."""
    from oracle import cpu_walk
    from tests import pyramid_walk as PW
    depth, color = golden["depth"], golden["color"]
    H, W = depth.shape[1:]
    frames = (7, 2, 7, 5)
    for level in (1, 2, 3):
        w, h = W >> level, H >> level
        inputs = FW.Inputs(None, depth, color, None, FW.stage_pyramid(level, w, h))
        for f in frames:
            d, c = inputs.staged_frame(f)
            assert d.shape == (h, w) and c.shape == (h, w, 3)
            assert np.array_equal(d, PW.downscale_median_excluding(depth[f], w, h))
            assert np.array_equal(c, PW.color_image_pyramid(color[f], level))
    for passes in (1, 2, 3):
        inputs = FW.Inputs(None, depth, color, None, FW.stage_median(passes))
        for f in frames:
            d, c = inputs.staged_frame(f)
            expect = depth[f]
            for _ in range(passes):
                expect = cpu_walk.median_filter_and_densify(expect)
            assert np.array_equal(d, expect) and np.array_equal(c, color[f])
            assert (d != 0).sum() > (depth[f] != 0).sum(), "the passes densify"
    inputs = FW.Inputs(None, depth, color, None)
    assert all(np.array_equal(inputs.staged_frame(f)[0], depth[f]) for f in frames)


def test_push_to_source_map_with_frames_left_out():
    """A relocalising session leaves its lost frames out: push p reads source frame sources[p], and its outlier
    neighbours are the K/2 pushes on either side, which skip the frames left out. Without relocalisation every frame is
    pushed, lost or not."""
    states = ["tracked"] * 6 + ["lost", "lost", "relocalised"] + ["tracked"] * 7
    sources = FW.pushed_sources(states)
    assert sources == [0, 1, 2, 3, 4, 5, 8, 9, 10, 11, 12, 13, 14, 15]
    assert FW.pushed_sources(states, held_out=False) == list(range(len(states)))
    pp = golden_params(load_golden())[0]
    assert pp.outlier_filtering_frame_count == 8
    inputs = FW.Inputs(None, None, None, pp, sources=sources)
    assert inputs.source(6) == 8
    assert inputs.others(4) == [3, 2, 1, 0, 5, 8, 9, 10]
    assert inputs.others(7) == [8, 5, 4, 3, 10, 11, 12, 13]
    # the caller extends the map while the session runs
    sources.append(16)
    assert inputs.source(10) == 12 and inputs.others(10) == [11, 10, 9, 8, 13, 14, 15, 16]
    assert FW.Inputs(None, None, None, pp).others(6) == [5, 4, 3, 2, 7, 8, 9, 10]
