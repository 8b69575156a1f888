"""The float64 restatement of the bilateral filter, outlier fusion and erosion (tests/preprocess_walk.py) against
the reference's recorded stages on the golden frames and against hand-built cases with closed-form answers."""
import itertools
import math

import numpy as np
import pytest

from tests import preprocess_walk as P
from tests.util import golden_camera, golden_params, other_frames


def golden_bilateral(golden, frame, pp):
    return P.Bilateral(golden["depth"][frame], pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor,
                       pp.bilateral_filter_radius_factor, int(pp.depth_scaling * pp.max_depth),
                       pp.depth_valid_region_radius)


def test_restatement_matches_reference_on_golden_frames(golden):
    """The reference's bilateral, outlier and erosion outputs of every golden frame satisfy the restatement: every
    clear pixel exact, every other one within its bound."""
    cam = golden_camera(golden)
    pp, _ = golden_params(golden)
    first, last = [int(v) for v in golden["frames"]]
    worst, shares, out_shares = 0.0, [], []
    for frame in range(first, last):
        b = golden_bilateral(golden, frame, pp)
        bad, frac, share = b.check(golden[f"f{frame}_bilateral"])
        assert bad == 0, f"frame {frame}: {bad} bilateral pixels off the restatement"
        worst, shares = max(worst, frac), shares + [share]
        others = [golden["depth"][f] for f in other_frames(frame, pp.outlier_filtering_frame_count)]
        o = P.Outlier(golden[f"f{frame}_bilateral"], cam, others, golden["others_TR_reference"][frame],
                      pp.outlier_filtering_depth_tolerance_factor, pp.outlier_filtering_required_inliers)
        wrong, out_share = o.check(golden[f"f{frame}_bilateral"], golden[f"f{frame}_outlier"])
        assert wrong == 0, f"frame {frame}: {wrong} outlier decisions off the restatement"
        assert (o.keep & o.clear).sum() > 0.8 * (golden[f"f{frame}_outlier"] != 0).sum()
        out_shares.append(out_share)
        assert np.array_equal(P.erode64(golden[f"f{frame}_outlier"], pp.depth_erosion_radius),
                              golden[f"f{frame}_erode"])
    assert worst <= 1.0
    print(f"golden frames: worst bilateral pixel uses {worst:.3f} of its bound; "
          f"{100 * max(shares):.1f} % of filtered pixels inside the rounding margin, "
          f"{100 * max(out_shares):.1f} % of outlier decisions inside theirs")


def test_bilateral_bound_resolves_a_wrong_tap_weight(golden):
    """The bound is far below what a 1 % change of the range weights moves: the restatement with sigma_v 1 % larger
    disagrees with the reference's output on clear pixels."""
    pp, _ = golden_params(golden)
    frame = int(golden["frames"][0])
    pp.bilateral_filter_sigma_depth_factor *= 1.01
    b = golden_bilateral(golden, frame, pp)
    assert b.check(golden[f"f{frame}_bilateral"])[0] > 100


def bilateral(raw, sigma_xy=3.0, sigma_v=0.05, factor=2.0, max_depth=15000, valid=1e6):
    return P.Bilateral(np.asarray(raw, np.uint16), sigma_xy, sigma_v, factor, max_depth, valid)


def test_constant_patch_returns_its_depth():
    b = bilateral(np.full((20, 24), 7777))
    assert b.active.all() and np.abs(b.value - 7777).max() < 1e-9
    assert b.clear.all() and (b.expected == 7777).all()
    assert b.taps[10, 12] == 113 and b.taps[0, 0] == sum(1 for dy, dx in P.disc_taps(6) if dy >= 0 and dx >= 0)


def test_depth_step_next_to_an_ignored_tap():
    """sigma_xy 1, radius factor 2: R = 2, 13 taps. Columns x <= 5 hold c, the rest c2, and one tap is 0: v is the
    two-level weighted mean with the ignored tap left out."""
    c, c2, sv = 2000, 2040, 0.05
    raw = np.full((9, 11), c, np.uint16)
    raw[:, 6:] = c2
    raw[3, 5] = 0
    b = bilateral(raw, sigma_xy=1.0, sigma_v=sv, factor=2.0)
    assert b.R == 2
    y, x = 4, 5
    num = den = 0.0
    for dy, dx in P.disc_taps(2):
        s = int(raw[y + dy, x + dx])
        if s == 0:
            continue
        w = math.exp(-(dx * dx + dy * dy) / 2.0 - (c - s) ** 2 / (2 * (c * P.f32(sv)) ** 2))
        num, den = num + w * s, den + w
    assert b.taps[y, x] == 12
    assert abs(b.value[y, x] - num / den) < 1e-9 and c < b.value[y, x] < c2
    assert b.expected[y, x] == math.floor(num / den + 0.5)
    assert not b.active[3, 5] and b.expected[3, 5] == 0


def test_max_depth_is_kept_and_one_above_is_cut():
    raw = np.full((7, 7), 3000, np.uint16)
    raw[3, 3], raw[3, 4] = 3000, 3001
    b = bilateral(raw, max_depth=3000)
    assert b.active[3, 3] and not b.active[3, 4] and b.expected[3, 4] == 0


def test_valid_region_circle_edge():
    """21 x 21, centre (10, 10), radius 5: d^2 = 25 is inside, 26 is not."""
    b = bilateral(np.full((21, 21), 4000), valid=5.0)
    assert b.active[10, 15] and b.active[14, 13] and b.active[10, 5]
    assert not b.active[11, 15] and not b.active[10, 16] and not b.active[16, 10]
    assert b.active.sum() == sum(1 for y in range(21) for x in range(21) if (x - 10) ** 2 + (y - 10) ** 2 <= 25)


def test_ignored_tap_instantiation_predicate():
    assert P.ignored_taps_vanish(0.05) and P.ignored_taps_vanish(0.0674)
    assert not P.ignored_taps_vanish(0.0675) and not P.ignored_taps_vanish(0.1) and not P.ignored_taps_vanish(0.5)


# Outlier fusion: fx = 128, cx = 0.5, depth 1024: p_x = 8 x, and a frame shifted by t_x projects pixel x to
# u = x + t_x / 8 + 0.5 exactly in float64.
EDGE_CAM = (16, 4, 128.0, 128.0, 0.5, 0.5)


def shifted(tx):
    m = np.zeros((3, 4), np.float32)
    m[:, :3] = np.eye(3)
    m[0, 3] = tx
    return m


def test_projection_on_the_image_edge():
    W, H = EDGE_CAM[:2]
    depth = np.full((H, W), 1024, np.uint16)
    other = np.full((H, W), 1024, np.uint16)
    cases = {4: (W - 1, False), 3: (W - 1, True), -12: (0, False), -11: (0, True), -4: (0, True)}
    for tx, (x, inside) in cases.items():
        o = P.Outlier(depth, EDGE_CAM, [other, other], [shifted(tx), shifted(tx)], 0.02)
        assert o.keep[1, x] == inside, (tx, x)
    # u = W and u = -1 lie on an edge: inside the margin; u = W - 1/8 and u = -7/8 are clear, and so is u = -0.5,
    # which truncates to column 0 with no edge near it
    assert not P.Outlier(depth, EDGE_CAM, [other] * 2, [shifted(4)] * 2, 0.02).clear[1, W - 1]
    assert not P.Outlier(depth, EDGE_CAM, [other] * 2, [shifted(-12)] * 2, 0.02).clear[1, 0]
    for tx, x in ((3, W - 1), (-11, 0), (-4, 0)):
        assert P.Outlier(depth, EDGE_CAM, [other] * 2, [shifted(tx)] * 2, 0.02).clear[1, x]


@pytest.mark.parametrize("required,kept", [(-1, False), (4, False), (3, True), (1, True)])
def test_required_inlier_count(required, kept):
    """Four identity frames, one of which holds a depth 3 % off: three agree."""
    W, H = EDGE_CAM[:2]
    depth = np.full((H, W), 1024, np.uint16)
    good, bad = depth.copy(), np.full((H, W), 1055, np.uint16)
    o = P.Outlier(depth, EDGE_CAM, [good, bad, good, good], [shifted(0)] * 4, 0.02, required)
    assert (o.ok_lo[:, 1:-1] == 3).all() and (o.ok_hi[:, 1:-1] == 3).all()
    assert (o.keep[:, 1:-1] == kept).all() and o.clear.all()


def test_tolerance_edges():
    """An other frame at ratio r of the depth agrees for r in [0.98, 1.02]; ratios within the margin of an edge are
    flagged, the rest are exact."""
    W, H = 64, 2
    cam = (W, H, 128.0, 128.0, 0.5, 0.5)
    depth = np.full((H, W), 10000, np.uint16)
    other = np.tile(np.arange(9790, 9790 + 2 * W * 5, 10)[:W].astype(np.uint16), (H, 1))
    o = P.Outlier(depth, cam, [other, other], [shifted(0)] * 2, 0.02)
    ratio = other[0].astype(np.float64) / 10000
    agree = (ratio >= 0.98) & (ratio <= 1.02)
    clear = o.clear[0]
    assert (o.keep[0][clear] == agree[clear]).all() and agree.any() and (~agree).any()
    assert not clear[np.abs(ratio - 0.98) < 1e-9].any() and not clear[np.abs(ratio - 1.02) < 1e-9].any()
    assert clear[np.abs(ratio - 1.0) < 0.019].all()


def test_erosion_and_border_copy():
    d = np.full((9, 10), 500, np.uint16)
    d[4, 6] = 0
    assert np.array_equal(P.erode64(d, 0)[1:-1, 1:-1], d[1:-1, 1:-1]) and not P.erode64(d, 0)[0].any()
    e1 = P.erode64(d, 1)
    assert e1[4, 4] == 500 and e1[3, 5] == 0 and e1[5, 7] == 0 and e1[1, 1] == 500 and e1[0, 1] == 0
    full = P.erode64(np.full((9, 10), 500, np.uint16), 3)
    assert full[3:6, 3:7].all() and np.count_nonzero(full) == 12
    assert not P.erode64(d, 3).any()   # every 7 x 7 window of the interior covers the hole
    assert not P.erode64(np.full((6, 6), 9, np.uint16), 3).any() and not P.erode64(np.full((2, 9), 9, np.uint16), 0).any()


def test_four_neighbours_and_isolated_pixels():
    d = np.zeros((5, 5), np.uint16)
    d[1:4, 1:4] = 7
    assert np.array_equal(P.four_neighbours(d), np.pad(np.ones((1, 1), bool), 2))
    n = P.neighbour_count(d)
    assert n[2, 2] == 8 and n[1, 1] == 3 and n[0, 0] == 1 and n[1, 2] == 5


def test_fused_tail_indices_stay_in_range_at_every_frame_size():
    """The shared-memory and guarded global indices of k_erode_normals_radii, restated for every size and erosion
    radius of the GPU frame-size sweep (tests/test_preprocess_fused_gpu.py) before any of them runs."""
    from tests.test_preprocess_fused_gpu import MAX_ERODE, SIZES, tail_index_ranges
    for (w, h), r in itertools.product(SIZES, range(MAX_ERODE + 1)):
        ranges = tail_index_ranges(w, h, r)
        assert ranges["sB (erosion centre)"][1] < ranges["sB (erosion centre)"][2]
    # radius 3 reads the first and the last row of the TMA box
    rows = tail_index_ranges(32, 16, 3)["sB (row validity)"]
    assert rows[0] // 48 == 0 and rows[1] // 48 == 25
