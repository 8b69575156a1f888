"""GPU parity tests: the product's sm_90a kernels (through the C ABI) against
  (1) the committed golden vectors (outputs of the reference's own kernels, tests/golden/),
  (2) the reference's kernels on the same seeded inputs: their recorded answers
      (tests/golden/oracle_answers.json, tests/golden/make_oracle_answers.py) or, where the
      oracle's state feeds the product frame by frame, the oracle run live (oracle/_ref), and
  (3) size-independent properties at the benchmark's full size.

Bar (north_star): integer / index work bit-exact, floats within 1e-4 relative. Where the
reference itself is not run-to-run deterministic (which of several supporting surfels wins a
pixel, float atomics; SURVEY §7 hard part 1) the contract is stated in the test.
"""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, SurfelError
from tests.util import (GOLDEN_DIR, INTEGRATE_ROWS, INVALID, NEIGHBOR_ROWS, SMOOTH_ROWS, check_state_invariants,
                        count_mismatch, digest, golden_camera, golden_params, link_stable_slots, load_npz_xz,
                        oracle_answers, other_frames, regularization_threshold, smooth_violations)

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def u16(h, w):
    return torch.zeros((h, w), dtype=torch.uint16, device="cuda")


def run_stages(lib, cam, pp, raw, others, mats, forced=None):
    """The five reference stages through `lib`. With `forced` (dict of oracle outputs) every
    stage consumes the oracle's previous stage instead of its own (teacher forcing)."""
    W, H, fx, fy, cx, cy = cam
    o = {}
    o["bilateral"] = u16(H, W)
    R.BilateralFilteringAndDepthCutoffCUDA(None, pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor, 0,
                                           pp.bilateral_filter_radius_factor, int(pp.depth_scaling * pp.max_depth),
                                           pp.depth_valid_region_radius, raw, o["bilateral"], lib=lib)
    src = forced or o
    o["outlier"] = u16(H, W)
    R.OutlierDepthMapFusionCUDA(None, pp.outlier_filtering_depth_tolerance_factor, src["bilateral"], fx, fy, cx, cy,
                                others, mats, o["outlier"], required_count=pp.outlier_filtering_required_inliers,
                                lib=lib)
    o["erode"] = u16(H, W)
    R.ErodeDepthMapCUDA(None, pp.depth_erosion_radius, src["outlier"], o["erode"], lib=lib)
    o["normals_depth"] = u16(H, W)
    o["normals"] = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
    R.ComputeNormalsAndDropBadPixelsCUDA(None, pp.observation_angle_threshold_deg, pp.depth_scaling, fx, fy, cx, cy,
                                         src["erode"], o["normals_depth"], o["normals"], lib=lib)
    o["pre_depth"] = u16(H, W)
    o["radius"] = torch.zeros((H, W), dtype=torch.float32, device="cuda")
    R.ComputePointRadiiAndRemoveIsolatedPixelsCUDA(None, pp.point_radius_extension_factor, pp.point_radius_clamp_factor,
                                                   pp.depth_scaling, fx, fy, cx, cy, src["normals_depth"], o["radius"],
                                                   o["pre_depth"], lib=lib)
    torch.cuda.synchronize()
    return o


STAGES = ("bilateral", "outlier", "erode", "normals_depth", "normals", "pre_depth", "radius")


def stage_digests(o):
    """Digests of the five stages' outputs (the radius only where the normals stage kept the pixel: elsewhere
    the reference leaves it unwritten)."""
    out = {k: digest(o[k].cpu().numpy()) for k in STAGES if k != "radius"}
    written = o["normals_depth"].cpu().numpy() != 0
    out["radius"] = digest(np.where(written, o["radius"].cpu().numpy().view(np.uint32), 0))
    return out


def assert_stages_match_answers(mine, key):
    """Every stage bit-exact against the reference's recorded answer for `key`."""
    want = oracle_answers()[key]
    got = stage_digests(mine)
    assert [k for k in STAGES if got[k] != want[k]] == [], f"{key}: stages differing from the reference"


def assert_stages_equal(mine, ref):
    for k in ("bilateral", "outlier", "erode", "normals_depth", "normals", "pre_depth"):
        assert count_mismatch(mine[k].cpu().numpy(), np.asarray(ref[k].cpu() if torch.is_tensor(ref[k]) else ref[k])) == 0, k
    nd = ref["normals_depth"]
    written = (nd.cpu().numpy() if torch.is_tensor(nd) else np.asarray(nd)) != 0
    rr = ref["radius"]
    assert count_mismatch(mine["radius"].cpu().numpy(), rr.cpu().numpy() if torch.is_tensor(rr) else np.asarray(rr),
                          written) == 0, "radius"


# ---------------------------------------------------------------------------------------
# depth pre-processing
# ---------------------------------------------------------------------------------------

def test_preprocess_stages_match_golden_bit_exact(golden, product):
    cam = golden_camera(golden)
    pp, _ = golden_params(golden)
    first, last = [int(v) for v in golden["frames"]]
    depth = dev(golden["depth"])
    for frame in range(first, last):
        others = [depth[f] for f in other_frames(frame, pp.outlier_filtering_frame_count)]
        forced = {k: dev(golden[f"f{frame}_{k}"]) for k in ("bilateral", "outlier", "erode", "normals_depth")}
        mine = run_stages(product, cam, pp, depth[frame], others, golden["others_TR_reference"][frame], forced)
        ref = {k: golden[f"f{frame}_{k}"] for k in ("bilateral", "outlier", "erode", "normals_depth", "normals",
                                                      "pre_depth", "radius")}
        assert_stages_equal(mine, ref)


def test_fused_preprocess_matches_golden_bit_exact(golden, product):
    W, H, fx, fy, cx, cy = golden_camera(golden)
    pp, _ = golden_params(golden)
    first, last = [int(v) for v in golden["frames"]]
    depth = dev(golden["depth"])
    rec = R.CUDASurfelReconstruction(int(golden["cap"][0]), W, H, fx, fy, cx, cy)
    for frame in range(first, last):
        others = [depth[f] for f in other_frames(frame, pp.outlier_filtering_frame_count)]
        d, n, r = u16(H, W), torch.zeros((H, W, 2), device="cuda"), torch.zeros((H, W), device="cuda")
        rec.preprocess(None, pp, depth[frame], others, golden["others_TR_reference"][frame], d, n, r)
        torch.cuda.synchronize()
        assert count_mismatch(d.cpu().numpy(), golden[f"f{frame}_pre_depth"]) == 0
        assert count_mismatch(n.cpu().numpy(), golden[f"f{frame}_normals"]) == 0
        written = golden[f"f{frame}_normals_depth"] != 0
        assert count_mismatch(r.cpu().numpy(), golden[f"f{frame}_radius"], written) == 0


RAGGED_SIZES = [(640, 480), (333, 201), (64, 48)]


def ragged_case(width, height):
    """Inputs of test_preprocess_live_oracle_ragged_sizes: (cam, pp, raw, others, mats, input digest)."""
    cam_ = S.Camera.tum(width, height) if (width, height) == (640, 480) else S.Camera(width, height, 525.0 * width / 640,
                                                                                      525.0 * width / 640, width / 2.0,
                                                                                      height / 2.0)
    st = S.make_stream(cam_, 10, stream_id=3, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam_.valid_region_radius()
    cam = (width, height, cam_.fx, cam_.fy, cam_.cx, cam_.cy)
    frame = 5
    others = [st.depth[f] for f in other_frames(frame, 8)]
    return cam, pp, st.depth[frame], others, st.others_TR_reference[frame], digest(st.depth.cpu().numpy())


@pytest.mark.parametrize("width,height", RAGGED_SIZES)
def test_preprocess_live_oracle_ragged_sizes(product, width, height):
    """Image sizes that are not multiples of the tile / vector width, against the reference's answers
    (every stage of the free-running chain bit-exact)."""
    cam, pp, raw, others, mats, inputs = ragged_case(width, height)
    key = f"preprocess/{width}x{height}"
    assert inputs == oracle_answers()[key]["inputs"], "the seeded input stream changed"
    assert_stages_match_answers(run_stages(product, cam, pp, raw, others, mats), key)


PREPROCESS_VARIANTS = ["required3of4", "erode0", "erode1", "erode3", "radius4", "clamp", "pitched", "all_invalid"]


def variant_case(variant):
    """Inputs of test_preprocess_variants_live_oracle: (cam, pp, raw, others, mats, input digest)."""
    cam_ = S.Camera.tum(320, 240)
    st = S.make_stream(cam_, 10, stream_id=5, device="cuda")
    W, H = 320, 240
    cam = (W, H, cam_.fx, cam_.fy, cam_.cx, cam_.cy)
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam_.valid_region_radius()
    frame, K = 5, 8
    raw = st.depth[frame]
    if variant == "required3of4":
        K = 4
        pp.outlier_filtering_frame_count, pp.outlier_filtering_required_inliers = 4, 3
    elif variant.startswith("erode"):
        pp.depth_erosion_radius = int(variant[-1])
    elif variant == "radius4":
        pp.bilateral_filter_sigma_xy = 2.0  # radius = int(2 * 2 + 0.5) = 4: generic-radius kernel
    elif variant == "clamp":
        pp.point_radius_clamp_factor = 1.2
    elif variant == "pitched":
        wide = torch.zeros((H, W + 24), dtype=torch.uint16, device="cuda")
        wide[:, :W] = raw
        raw = wide[:, :W]  # pitch != W * 2
    elif variant == "all_invalid":
        raw = torch.zeros_like(raw)
    others = [st.depth[f] for f in other_frames(frame, K)]
    mats = S.others_TR_reference(st.global_T_frame.astype(np.float64), pp.depth_scaling, K)[frame]
    return cam, pp, raw, others, mats, digest(st.depth.cpu().numpy())


@pytest.mark.parametrize("variant", PREPROCESS_VARIANTS)
def test_preprocess_variants_live_oracle(product, variant):
    cam, pp, raw, others, mats, inputs = variant_case(variant)
    key = f"preprocess_variant/{variant}"
    assert inputs == oracle_answers()[key]["inputs"], "the seeded input stream changed"
    mine = run_stages(product, cam, pp, raw, others, mats)
    assert_stages_match_answers(mine, key)
    if variant == "all_invalid":
        assert not mine["pre_depth"].cpu().numpy().any()


# ---------------------------------------------------------------------------------------
# Integrate()
# ---------------------------------------------------------------------------------------

DETERMINISTIC_RASTERS = ("first_surfel_depth", "supporting_surfel_counts", "conflicting_surfels",
                         "new_surfel_flag_vector", "new_surfel_indices")


# The nondeterministic rows are held to the reference's OWN run-to-run difference (oracle B against oracle A on the
# same frame): at most ENVELOPE_FACTOR times that, plus a floor for the frames where two oracle runs happen to agree
# almost exactly (the first integrated frame: all surfels come from one creation sweep, the reference's race is
# nearly reproducible there and any other resolution differs by a few units). See DESIGN.md section 4.
ENVELOPE_FACTOR = 2


def envelope_floors(n_before):
    """(merge flags / merge count, neighbour-link rows)"""
    return 12, max(24, n_before // 200)


def envelope_limit(env, floor):
    """ENVELOPE_FACTOR x the oracle's own difference, plus four standard deviations of that count (one oracle pair is
    a single draw: a count of ~50 differing flags scatters by +-7 from run to run), plus the floor."""
    return ENVELOPE_FACTOR * env + 4.0 * float(np.sqrt(max(env, 1))) + floor


# Number of extra oracle runs (B) a live-oracle test measures the reference's envelope with. A single B draw can
# land low (two runs of the reference happen to agree unusually well on a frame), and a test family with hundreds of
# envelope checks then fails now and then on an unchanged build; the envelope is the largest of several draws.
ORACLE_B_RUNS = 3


def race_envelope(states_b, state_a, n_before):
    """What further runs of the oracle (B) differ from the first (A) in, on the race-bound rows of the slots that
    existed before the frame: (differing merge flags, |merge count difference|, differing neighbour-link rows), each
    the largest over the B runs. The product is held to a multiple of this (compare_integrate)."""
    rows_a, _, merges_a = state_a
    nb = list(NEIGHBOR_ROWS)
    out = (0, 0, 0)
    for rows_b, _, merges_b in states_b:
        flags = int(((rows_b[7, :n_before] < 0) != (rows_a[7, :n_before] < 0)).sum())
        links = int((rows_b[nb, :n_before].view(np.uint32) != rows_a[nb, :n_before].view(np.uint32)).any(axis=0).sum())
        out = tuple(max(a, b) for a, b in zip(out, (flags, abs(int(merges_b) - int(merges_a)), links)))
    return out


def smooth_floor(n_before):
    """Floor of the smooth-position envelope: a neighbour link that differs (link floor of envelope_floors) moves the
    smooth positions of the up to four slots it touches through their accumulated gradients."""
    return max(24, n_before // 200)


# Measured (H100 80GB HBM3, 700 W, October 2026; three full suite runs, 573 frames with an envelope): the product broke
# the smooth bound on at most 281 of 48 624 link-stable slots where the B runs broke it on up to 461 of the same set;
# the largest product count relative to its oracle figure was 253 against 198 (17 100 slots). Golden frames: 0, 8, 22
# and 27 of 8 206 - 11 130 slots (<= 0.3 %).
# Without a second oracle run (golden vectors) at most this fraction of the link-stable slots may break the smooth
# tolerance: the bound of test_smooth_positions_close_to_oracle.
SMOOTH_GOLDEN_FRACTION = 0.02


def compare_smooth(rows_m, rows_r, frame_index, window, iterations, rows_b=(), n_before=0, label=""):
    """Smooth positions (rows 3-5) after a regularisation that started from the same state in both runs.
    - outside the window (int(stamp) < int(frame_index - window), stamps and merge flags equal): bit-exact; no
      sweep moves them, so both still hold the position they started from (the library's partial sweep has to
      carry these over between its two record buffers);
    - `iterations` == 0 (copy only, no float atomics): bit-exact for every in-window slot whose position rows,
      stamp and merge flag agree;
    - otherwise, on the link-stable slots (util.link_stable_slots): |delta| <= 1e-4 |p| + 1e-5 m per component
      except for at most envelope_limit(env, smooth_floor) slots, env = the most slots of that set on which a further
      oracle run (`rows_b`, a list) breaks the same bound against the first, or SMOOTH_GOLDEN_FRACTION of the set
      without one. The set is taken from the product against oracle A, so env also counts the slots whose links
      differ between the two oracle runs."""
    stamps_m, stamps_r = rows_m[18].view(np.int32), rows_r[18].view(np.int32)
    same = ((rows_m[7] < 0) == (rows_r[7] < 0)) & (stamps_m == stamps_r)
    outside = stamps_m < regularization_threshold(frame_index, window)
    smooth_bits = lambda rows: rows[list(SMOOTH_ROWS)].view(np.uint32)
    differs = np.any(smooth_bits(rows_m) != smooth_bits(rows_r), axis=0)
    assert int((differs & same & outside).sum()) == 0, f"{label}smooth positions outside the regularisation window"
    if iterations == 0:
        same_position = np.all(rows_m[0:3].view(np.uint32) == rows_r[0:3].view(np.uint32), axis=0)
        assert int((differs & same & ~outside & same_position).sum()) == 0, f"{label}copy-only smooth positions"
        return
    stable = link_stable_slots(rows_m, rows_r)
    got = smooth_violations(rows_m, rows_r, stable)
    if not len(rows_b):
        limit = SMOOTH_GOLDEN_FRACTION * int(stable.sum())
        env = None
    else:
        env = max(smooth_violations(rows, rows_r, stable) for rows in rows_b)
        limit = envelope_limit(env, smooth_floor(n_before))
    print(f"{label}smooth: {got} of {int(stable.sum())} link-stable slots outside 1e-4 |p| + 1e-5 m "
          f"(oracle B: {env}, window {int((~outside).sum())}, n = {rows_m.shape[1]})")
    assert got <= limit, (label, got, env, int(stable.sum()))


def link_attribution(walk, mine_rasters, ref_rasters, rows_m, rows_r, n_before):
    """Where the neighbour links of the product and oracle A may legitimately differ. `walk` = the frame's inputs
    (rows before the frame, frame index, (fx, fy, cx, cy), frame_T_global, pre-blend depth, normals, IntegrateParams).
    The CPU walk (oracle/cpu_walk.c) recomputes every pixel's supporter set from the state before the frame; the
    product's supporting surfel of every contested pixel must be a member of it (a legal race outcome). A slot's links
    may then differ only if it has an association within 3 pixels of a pixel the two runs resolved differently (the
    integration can move a surfel by a pixel before its neighbourhood is read, as in test_round2_gpu), or if it or one
    of its link targets merged differently. Returns (differing link rows outside that set, slots in it)."""
    if n_before == 0:
        return 0, 0   # an empty cloud: no slot had links, and no pixel had a supporter
    from tests.test_round2_gpu import supporter_sets
    from oracle import cpu_walk
    from scipy import ndimage
    fx, fy, cx, cy = walk["camera"]
    ip = walk["ip"]
    _, ev_p, ev_k = cpu_walk.associate_events(walk["rows"], walk["frame_index"], fx, fy, cx, cy, walk["frame_T_global"],
                                              walk["depth"], walk["normals"], ip.sensor_noise_factor,
                                              ip.normal_compatibility_threshold_deg, ip.depth_scaling)
    sets = supporter_sets(ev_p, ev_k)
    cnt = ref_rasters["supporting_surfel_counts"].reshape(-1)
    sup_m, sup_r = mine_rasters["supporting_surfels"].reshape(-1), ref_rasters["supporting_surfels"].reshape(-1)
    contested = np.flatnonzero(cnt > 1)
    checked = outside = 0
    for p in contested:
        s = sets.get(int(p))
        if s is None or len(s) != cnt[p]:
            continue  # CPU and GPU floats disagree on a borderline gate: not a statement about the winner
        checked += 1
        outside += int(sup_m[p] not in s)
    assert outside == 0 and checked >= 0.9 * len(contested), ("supporting surfel outside the supporter set",
                                                              checked, len(contested), outside)
    H, W = ref_rasters["supporting_surfel_counts"].shape
    resolved = ((cnt > 1) & (sup_m != sup_r)).reshape(H, W)
    near = ndimage.binary_dilation(resolved, structure=np.ones((3, 3), bool), iterations=3).reshape(-1)
    attributable = np.zeros(n_before, bool)
    slots = (ev_k[near[ev_p]] & 0x7FFFFFFF).astype(np.int64)
    attributable[slots[slots < n_before]] = True
    nb = list(NEIGHBOR_ROWS)
    links_m, links_r = rows_m[nb, :n_before].view(np.uint32), rows_r[nb, :n_before].view(np.uint32)
    bad = np.flatnonzero((rows_m[7, :n_before] < 0) != (rows_r[7, :n_before] < 0))
    attributable |= np.isin(np.arange(n_before), bad) | np.isin(links_m, bad).any(axis=0) | np.isin(links_r, bad).any(axis=0)
    differ = (links_m != links_r).any(axis=0)
    return int((differ & ~attributable).sum()), int(attributable.sum())


def compare_integrate(mine_rasters, mine_depth, mine_state, ref_rasters, ref_depth, ref_state, n_before, states_b=(),
                      ip=None, frame_index=None, walk=None):
    """Contract for one teacher-forced Integrate():
    - min-depth raster, supporting counts, conflicting surfels, new-surfel flags + scan indices,
      surfel count: bit-exact;
    - blended depth: bit-exact except where the float-atomic depth sum of a border pixel rounds
      differently (<= 5 pixels per frame, 1 LSB each; the reference differs from itself likewise);
    - supporting surfel: same pixel set; identical where one surfel supports the pixel;
      otherwise one of the supporters (the reference takes whichever atomicCAS arrives first);
    - depth sums: 1e-6 relative (float atomics);
    - per-surfel attributes written by the integration (position, confidence, radius, normal,
      stamps, colour) bit-exact for every surfel whose merge decision agrees (merging reads the
      supporting surfel, so it inherits its nondeterminism): with `states_b` (the states of further
      oracle runs; race_envelope) the differing merge flags and the merge-count difference stay within
      ENVELOPE_FACTOR x the reference's own run-to-run difference (+ a floor); without them (golden vectors: a
      single recorded run) within small absolute bounds;
    - neighbour links: with `walk` (the frame's inputs, link_attribution) every supporting surfel of a contested
      pixel is one of the pixel's supporters, and a link differs only on slots next to a pixel the two runs resolved
      differently or touched by a differing merge (up to the tolerance of test_round2_gpu's exact-link check);
      without it, the differing link rows stay within the envelope (+ a floor fitted at VGA);
    - smooth positions: compare_smooth with the frame's regularisation window and sweep count (`ip`,
      `frame_index`): bit-exact outside the window and for copy-only frames, otherwise 1e-4 relative
      (+ 1e-5 m) on the slots whose own and neighbours' links and merge flags agree, up to the envelope."""
    envelope = race_envelope(states_b, ref_state, n_before) if len(states_b) else None
    for k in DETERMINISTIC_RASTERS:
        assert count_mismatch(mine_rasters[k], ref_rasters[k]) == 0, k
    depth_diff = np.abs(mine_depth.astype(np.int32) - ref_depth.astype(np.int32))
    assert (depth_diff != 0).sum() <= 5 and depth_diff.max() <= 1, "blended depth"
    sup_m, sup_r, cnt = mine_rasters["supporting_surfels"], ref_rasters["supporting_surfels"], \
        ref_rasters["supporting_surfel_counts"]
    assert np.array_equal(sup_m == INVALID, sup_r == INVALID)
    assert count_mismatch(sup_m, sup_r, cnt == 1) == 0
    s_m, s_r = mine_rasters["supporting_surfel_depth_sums"], ref_rasters["supporting_surfel_depth_sums"]
    assert np.allclose(s_m, s_r, rtol=1e-6, atol=0)
    rows_m, n_m, merges_m = mine_state
    rows_r, n_r, merges_r = ref_state
    assert n_m == n_r, "surfels_size()"
    same_merge = (rows_m[7] < 0) == (rows_r[7] < 0)
    nb = list(NEIGHBOR_ROWS)
    link_rows_differ = int((rows_m[nb, :n_before].view(np.uint32) != rows_r[nb, :n_before].view(np.uint32)).any(axis=0).sum())
    if envelope is not None:
        env_flags, env_count, env_links = envelope
        print(f"envelope: merge flags {int((~same_merge).sum())} vs {env_flags}, merge count {abs(int(merges_m) - int(merges_r))} vs "
              f"{env_count}, link rows {link_rows_differ} vs {env_links} (n = {n_before})")
        flag_floor, link_floor = envelope_floors(n_before)
        assert (~same_merge).sum() <= envelope_limit(env_flags, flag_floor), ((~same_merge).sum(), env_flags)
        # (two oracle runs can differ on dozens of flags and still count the same number of merges: the count
        #  envelope is the larger of the two figures)
        assert abs(int(merges_m) - int(merges_r)) <= envelope_limit(max(env_count, env_flags), flag_floor), (merges_m, merges_r, env_count, env_flags)
        if walk is None:
            assert link_rows_differ <= envelope_limit(env_links, link_floor), (link_rows_differ, env_links)
        else:
            unexplained, attributable = link_attribution(walk, mine_rasters, ref_rasters, rows_m, rows_r, n_before)
            print(f"links: {unexplained} differing rows away from differently resolved pixels and merges "
                  f"({attributable} slots near them)")
            assert unexplained <= 2 * env_links // 10 + 4, (unexplained, env_links)
    else:
        assert (~same_merge).sum() <= max(20, 0.004 * n_r), "merge decisions differ only inside the reference's envelope"
        assert abs(int(merges_m) - int(merges_r)) <= max(20, 0.004 * n_r)
        assert link_rows_differ <= max(40, 0.04 * n_before)
    # a blended-depth pixel that rounds differently (see above) feeds up to a few surfels
    allowed = 4 * int((depth_diff != 0).sum())
    for row in INTEGRATE_ROWS:
        assert count_mismatch(rows_m[row], rows_r[row], same_merge) <= allowed, f"row {row}"
    check_state_invariants(rows_m, n_m)
    assert ip is not None and frame_index is not None, "the smooth-position contract needs the frame's parameters"
    compare_smooth(rows_m, rows_r, frame_index, ip.regularization_frame_window_size,
                   ip.regularization_iterations_per_integration_iteration,
                   rows_b=[state[0] for state in states_b], n_before=n_before, label=f"frame {frame_index}: ")


def test_integrate_teacher_forced_against_golden(golden, product):
    W, H, fx, fy, cx, cy = golden_camera(golden)
    pp, ip = golden_params(golden)
    first, last = [int(v) for v in golden["frames"]]
    rec = R.CUDASurfelReconstruction(int(golden["cap"][0]), W, H, fx, fy, cx, cy)
    color = dev(golden["color"])
    for frame in range(first, last):
        if frame > first:
            n_prev, merges_prev = [int(v) for v in golden[f"f{frame - 1}_counts"]]
            rec.load_state(golden[f"f{frame - 1}_state"], merges_prev)
        else:
            n_prev = 0
        d = dev(golden[f"f{frame}_pre_depth"])
        rec.integrate(None, frame, ip, d, dev(golden[f"f{frame}_normals"]), dev(golden[f"f{frame}_radius"]),
                      color[frame], golden["global_T_frame"][frame], golden["frame_T_global"][frame])
        torch.cuda.synchronize()
        ref_rasters = {k: golden[f"f{frame}_{k}"] for k in DETERMINISTIC_RASTERS + (
            "supporting_surfels", "supporting_surfel_depth_sums")}
        n_r, merges_r = [int(v) for v in golden[f"f{frame}_counts"]]
        compare_integrate(rec.download_rasters(), d.cpu().numpy(), rec.dump_state(), ref_rasters,
                          golden[f"f{frame}_blended_depth"], (golden[f"f{frame}_state"], n_r, merges_r), n_prev, ip=ip,
                          frame_index=frame)
        assert rec.surfels_size() == n_r


# Cameras of the live-oracle cases: intrinsics in the pixel-corner convention, and the depth scaling of the stream,
# the pre-processing and the integration.
LIVE_CAMERAS = {
    "tum": (S.Camera.tum(640, 480), 5000.0),
    "tum_fr1": (S.Camera(640, 480, 517.3, 516.5, 319.1, 255.8), 5000.0),    # TUM RGB-D fr1 calibration
    "icl_nuim": (S.Camera(640, 480, 481.2, -480.0, 320.0, 240.0), 5000.0),  # ICL-NUIM: negative fy
    "odd": (S.Camera(333, 201, 290.0, 305.0, 171.3, 96.2), 5000.0),        # odd size, fx != fy, off-centre
    "mm": (S.Camera.tum(320, 240), 1000.0),                                 # depth in millimetres
}

# case: (camera, IntegrateParams overrides). The first six are the TUM-camera variants; the parameter cases run
# the odd camera, where every projection also has fx != fy and a width that is not a multiple of 16 (k_blend's
# scalar loads and stores).
LIVE_CASES = {
    "default": ("tum", {}),
    "no_blending": ("tum", {"do_blending": 0}),
    "reg0": ("tum", {"regularization_iterations_per_integration_iteration": 0}),
    "reg2": ("tum", {"regularization_iterations_per_integration_iteration": 2}),
    "window20": ("tum", {"surfel_integration_active_window_size": 2, "regularization_frame_window_size": 2}),
    "blend_radius5": ("tum", {"measurement_blending_radius": 5}),
    "tum_fr1": ("tum_fr1", {}),
    "icl_nuim": ("icl_nuim", {}),
    "odd": ("odd", {}),
    "mm": ("mm", {}),
    "sensor_noise0.02": ("odd", {"sensor_noise_factor": 0.02}),
    "max_confidence2": ("odd", {"max_surfel_confidence": 2.0}),
    "normal_threshold20": ("odd", {"normal_compatibility_threshold_deg": 20.0}),
    "weight2": ("odd", {"regularizer_weight": 2.0}),
    "weight40": ("odd", {"regularizer_weight": 40.0}),
    "radius_factor1.5": ("odd", {"radius_factor_for_regularization_neighbors": 1.5}),
    "radius_factor3": ("odd", {"radius_factor_for_regularization_neighbors": 3.0}),
    "blend_radius1": ("odd", {"measurement_blending_radius": 1}),     # <= 2: no iteration of the blending loop
    "blend_radius2": ("odd", {"measurement_blending_radius": 2}),
    "blend_radius24": ("odd", {"measurement_blending_radius": 24}),
    "pitched": ("odd", {}),
}


def live_case(case):
    """(camera, stream, PreprocessParams, IntegrateParams) of test_integrate_teacher_forced_live_oracle."""
    cam_name, overrides = LIVE_CASES[case]
    cam_, scale = LIVE_CAMERAS[cam_name]
    st = S.make_stream(cam_, 13, stream_id=11, depth_scaling=scale, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam_.valid_region_radius()
    pp.depth_scaling = scale
    ip = IntegrateParams.defaults()
    ip.depth_scaling = scale
    for k, v in overrides.items():
        setattr(ip, k, v)
    return cam_, st, pp, ip


CANARY16 = 0xBEEF


def pitched_inputs(d, n, r, c):
    """Views of copies of the four Integrate() inputs inside wider buffers: the depth view starts 2 bytes into its
    row (not 16-byte aligned: k_blend's scalar path), the others one or more pixels in. Returns (views, wide depth)."""
    H, W = d.shape
    wide_d = torch.full((H, W + 24), CANARY16, dtype=torch.int32, device="cuda").to(torch.uint16)
    wide_n = torch.full((H, W + 8, 2), float("nan"), device="cuda")
    wide_r = torch.full((H, W + 16), float("nan"), device="cuda")
    wide_c = torch.full((H, W + 5, 3), 77, dtype=torch.uint8, device="cuda")
    views = (wide_d[:, 1:1 + W], wide_n[:, 1:1 + W], wide_r[:, 3:3 + W], wide_c[:, 2:2 + W])
    for v, src in zip(views, (d, n, r, c)):
        v.copy_(src)
    assert views[0].data_ptr() % 16 == 2
    return views, wide_d


def preprocess_outputs(rec, pp, st, frame, H, W):
    """rec.preprocess of one stream frame into fresh buffers (radius pre-filled with NaN, so that the pixels the call
    writes can be told apart)."""
    others = [st.depth[f] for f in other_frames(frame, pp.outlier_filtering_frame_count)]
    d, n = u16(H, W), torch.zeros((H, W, 2), device="cuda")
    r = torch.full((H, W), float("nan"), device="cuda")
    rec.preprocess(None, pp, st.depth[frame], others, st.others_TR_reference[frame], d, n, r)
    return d, n, r


@pytest.mark.parametrize("case", list(LIVE_CASES))
def test_integrate_teacher_forced_live_oracle(product, reference, case):
    """Several frames, product re-synchronised to the oracle's state before every frame, on the cameras of real
    datasets (anisotropic, negative fy, odd size, millimetre depth) and non-default Integrate() parameters. The
    product's own pre-processing of the same frame is held to the oracle's bit for bit on the way."""
    cam_, st, pp, ip = live_case(case)
    W, H = cam_.width, cam_.height
    make = lambda lib=None: R.CUDASurfelReconstruction(600_000, W, H, cam_.fx, cam_.fy, cam_.cx, cam_.cy, lib=lib)
    rec_p, rec_r = make(), make(reference)
    recs_b = [make(reference) for _ in range(ORACLE_B_RUNS)]      # the oracle's own envelope
    rec_q = make() if case == "pitched" else None                  # packed inputs, against the pitched ones
    first, last = st.integrated_range()
    for frame in range(first, last):
        d0, n0, r0 = preprocess_outputs(rec_r, pp, st, frame, H, W)
        dq, nq, rq = preprocess_outputs(rec_p, pp, st, frame, H, W)
        torch.cuda.synchronize()
        assert count_mismatch(dq.cpu().numpy(), d0.cpu().numpy()) == 0, "pre-processed depth"
        assert count_mismatch(nq.cpu().numpy(), n0.cpu().numpy()) == 0, "normals"
        written = ~np.isnan(r0.cpu().numpy())
        assert written.any() and count_mismatch(rq.cpu().numpy(), r0.cpu().numpy(), written) == 0, "radius"
        r0 = torch.nan_to_num(r0, nan=0.0)
        rows, n_before, merges = rec_r.dump_state()
        for rec in [rec_p] + recs_b + ([rec_q] if rec_q else []):
            rec.load_state(rows, merges)
        dp, dr = d0.clone(), d0.clone()
        inputs_p = (dp, n0, r0, st.color[frame])
        if rec_q is not None:
            inputs_p, wide_d = pitched_inputs(dp, n0, r0, st.color[frame])
            dq = d0.clone()
            rec_q.integrate(None, frame, ip, dq, n0, r0, st.color[frame], st.global_T_frame[frame],
                            st.frame_T_global[frame])
        rec_p.integrate(None, frame, ip, *inputs_p, st.global_T_frame[frame], st.frame_T_global[frame])
        for rec, d in [(rec_r, dr)] + [(rec_b, d0.clone()) for rec_b in recs_b]:
            rec.integrate(None, frame, ip, d, n0, r0, st.color[frame], st.global_T_frame[frame], st.frame_T_global[frame])
        torch.cuda.synchronize()
        if rec_q is not None:
            wide = wide_d.cpu().numpy()
            assert (wide[:, 0] == CANARY16).all() and (wide[:, W + 1:] == CANARY16).all(), "padding written"
            dp = inputs_p[0]
            compare_product_runs(rec_p, dp.cpu().numpy(), rec_q, dq.cpu().numpy())
        state_p, state_r = rec_p.dump_state(), rec_r.dump_state()
        compare_integrate(rec_p.download_rasters(), dp.cpu().numpy(), state_p, rec_r.download_rasters(),
                          dr.cpu().numpy(), state_r, n_before, states_b=[rec.dump_state() for rec in recs_b], ip=ip,
                          frame_index=frame, walk=frame_walk(rows, frame, cam_, st, d0, n0, ip))
        assert rec_p.surfel_count() == rec_p.surfels_size() - state_p[2]
    if case == "max_confidence2":
        assert state_p[0][6].max() == 2.0, "the confidence clamp was reached"


def frame_walk(rows, frame_index, cam_, st, depth, normals, ip, stream_frame=None):
    """The inputs link_attribution recomputes a frame's supporter sets from (`depth`, `normals`: pre-blend tensors)."""
    f = frame_index if stream_frame is None else stream_frame
    return {"rows": rows, "frame_index": frame_index, "camera": (cam_.fx, cam_.fy, cam_.cx, cam_.cy),
            "frame_T_global": st.frame_T_global[f], "depth": depth.cpu().numpy(), "normals": normals.cpu().numpy(),
            "ip": ip}


def compare_product_runs(rec_a, depth_a, rec_b, depth_b):
    """Two product runs of one Integrate() on the same state and inputs. Everything but the float-atomic depth sums
    is deterministic in the product: rasters bit-equal, blended depth and the integrated rows bit-equal up to the
    pixels whose depth sum rounds differently (as compare_integrate)."""
    ras_a, ras_b = rec_a.download_rasters(), rec_b.download_rasters()
    for k in DETERMINISTIC_RASTERS + ("supporting_surfels",):
        assert count_mismatch(ras_a[k], ras_b[k]) == 0, k
    depth_diff = np.abs(depth_a.astype(np.int32) - depth_b.astype(np.int32))
    assert (depth_diff != 0).sum() <= 5 and depth_diff.max() <= 1, "blended depth"
    (rows_a, n_a, m_a), (rows_b, n_b, m_b) = rec_a.dump_state(), rec_b.dump_state()
    assert (n_a, m_a) == (n_b, m_b)
    for row in INTEGRATE_ROWS + NEIGHBOR_ROWS:
        assert count_mismatch(rows_a[row], rows_b[row]) <= 4 * int((depth_diff != 0).sum()), f"row {row}"


def test_smooth_positions_close_to_oracle(golden, product):
    """Regularised positions after a teacher-forced Integrate() (golden vectors: the reference's state before
    each frame and its pre-processed inputs): 1e-4 relative (+1e-5 m absolute) against the reference's state
    for surfels whose neighbour links and merge status agree; float atomics make the reference itself differ
    at this level."""
    W, H, fx, fy, cx, cy = golden_camera(golden)
    _, ip = golden_params(golden)
    first, last = [int(v) for v in golden["frames"]]
    rec = R.CUDASurfelReconstruction(int(golden["cap"][0]), W, H, fx, fy, cx, cy)
    color = dev(golden["color"])
    for frame in range(first, last):
        if frame > first:
            rec.load_state(golden[f"f{frame - 1}_state"], int(golden[f"f{frame - 1}_counts"][1]))
        rec.integrate(None, frame, ip, dev(golden[f"f{frame}_pre_depth"]), dev(golden[f"f{frame}_normals"]),
                      dev(golden[f"f{frame}_radius"]), color[frame], golden["global_T_frame"][frame],
                      golden["frame_T_global"][frame])
    torch.cuda.synchronize()
    rm, n, _ = rec.dump_state()
    rr, n2 = golden[f"f{last - 1}_state"], int(golden[f"f{last - 1}_counts"][0])
    assert n == n2
    nb = list(NEIGHBOR_ROWS)
    agree = np.all(rm[nb].view(np.uint32) == rr[nb].view(np.uint32), axis=0) & ((rm[7] < 0) == (rr[7] < 0))
    # neighbours of agreeing surfels may themselves disagree and shift the gradient: allow 2 % outliers
    close = np.all(np.isclose(rm[list(SMOOTH_ROWS)], rr[list(SMOOTH_ROWS)], rtol=1e-4, atol=1e-5), axis=0)
    assert (close | ~agree).mean() > 0.98


def golden_final_state(golden):
    """Input of the hand-off tests: the reference's state after the last golden frame (rows, n, merges, frame)."""
    last = int(golden["frames"][1])
    n, merges = [int(v) for v in golden[f"f{last - 1}_counts"]]
    return golden[f"f{last - 1}_state"], n, merges, last


def golden_reconstruction(golden, lib=None):
    W, H, fx, fy, cx, cy = golden_camera(golden)
    return R.CUDASurfelReconstruction(int(golden["cap"][0]), W, H, fx, fy, cx, cy, lib=lib)


def handoff_outputs(rec, frame_index, n):
    """TransferAllToCPU + ExportVertices of the current state: (digests, transfer buffers, exported positions)."""
    bufs = rec.TransferAllToCPU(None, frame_index)
    pos = torch.zeros(3 * n, dtype=torch.float32, device="cuda")
    col = torch.zeros(3 * n, dtype=torch.uint8, device="cuda")
    rec.ExportVertices(None, pos, col)
    torch.cuda.synchronize()
    pos, col = pos.cpu().numpy(), col.cpu().numpy()
    out = {k: digest(v[:n]) for k, v in bufs.items() if k.endswith("_buffer")}
    out.update(surfel_count=int(bufs["surfel_count"]), export_positions=digest(pos), export_colors=digest(col))
    return out, bufs, pos


def regularized_row_digests(rows):
    """The rows Regularize() must leave bit-exact (everything it may change is a smooth position)."""
    return {str(row): digest(rows[row].view(np.uint32)) for row in INTEGRATE_ROWS + NEIGHBOR_ROWS}


def test_regularize_transfer_export_against_oracle(golden, product):
    """Regularize(), TransferAllToCPU and ExportVertices on the reference's state after the golden frames,
    against what the reference's kernels answer on the same state (tests/golden/make_oracle_answers.py)."""
    rows, n, merges, last = golden_final_state(golden)
    ip = IntegrateParams.defaults()
    answers = oracle_answers()["golden_handoff"]
    assert digest(rows) == answers["inputs"]
    rec_p = golden_reconstruction(golden)
    rec_p.load_state(rows, merges)
    assert rec_p.surfels_size() == n and rec_p.surfel_count() == n - merges
    # TransferAllToCPU (the CUDASurfelBuffersCPU arrays) and ExportVertices: bit-exact
    got, bufs, pos = handoff_outputs(rec_p, last, n)
    assert got["surfel_count"] == n
    assert [k for k in got if got[k] != answers["handoff"][k]] == [], "hand-off outputs differing from the reference"
    assert count_mismatch(bufs["surfel_x_buffer"][:n], rows[3]) == 0, "x buffer carries the SMOOTH position"
    assert np.isnan(pos.reshape(-1, 3)[rows[7] < 0]).all(), "merged surfels export NaN positions"
    # Regularize(): identical inputs, float-atomic accumulation order differs -> 1e-4 relative
    rec_p.Regularize(None, last, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors,
                     ip.regularization_frame_window_size)
    torch.cuda.synchronize()
    rm = rec_p.dump_state()[0]
    smooth_r = load_npz_xz(GOLDEN_DIR / "oracle_regularized_smooth.npz.xz")["smooth"]
    assert np.allclose(rm[list(SMOOTH_ROWS)], smooth_r, rtol=1e-4, atol=1e-6)
    got = regularized_row_digests(rm)
    assert [r for r in got if got[r] != answers["regularized_rows"][r]] == [], \
        "integrated rows and neighbour links (far-neighbour pruning) are exact"


# ---------------------------------------------------------------------------------------
# edge cases and properties
# ---------------------------------------------------------------------------------------

def test_empty_cloud_and_empty_frame(product):
    """First frame on an empty cloud creates one surfel per valid interior pixel; an all-invalid
    frame creates nothing and changes nothing."""
    W, H = 96, 64
    rec = R.CUDASurfelReconstruction(50_000, W, H, 80.0, 80.0, 48.0, 32.0)
    ip = IntegrateParams.defaults()
    depth = torch.zeros((H, W), dtype=torch.int32)
    depth[8:40, 10:70] = 5000
    d = depth.to(torch.uint16).cuda()
    normals = torch.zeros((H, W, 2), device="cuda")
    radius = torch.full((H, W), 1e-4, device="cuda")
    color = torch.full((H, W, 3), 128, dtype=torch.uint8, device="cuda")
    pose = np.eye(4, dtype=np.float32)[:3]
    rec.integrate(None, 0, ip, d.clone(), normals, radius, color, pose)
    assert rec.surfels_size() == 32 * 60 and rec.surfel_count() == 32 * 60
    ras = rec.download_rasters()
    flags = ras["new_surfel_flag_vector"].reshape(-1)
    assert np.array_equal(ras["new_surfel_indices"].reshape(-1), np.cumsum(flags) - flags), "stable raster-order scan"
    rows, n, _ = rec.dump_state()
    assert np.all(rows[17].view(np.uint32) == 0) and np.allclose(rows[2], 1.0, atol=1e-6)
    check_state_invariants(rows, n)
    before = rows.copy()
    rec.integrate(None, 1, ip, torch.zeros((H, W), dtype=torch.uint16, device="cuda"), normals, radius, color, pose)
    rows2, n2, _ = rec.dump_state()
    assert n2 == n
    for row in INTEGRATE_ROWS:
        assert count_mismatch(before[row], rows2[row]) == 0


def test_capacity_overflow_is_reported(product):
    """The reference never checks the cap (SURVEY §5: it would write out of bounds); the product
    drops the frame's new surfels and reports SM_ERR_CAPACITY."""
    W, H = 96, 64
    rec = R.CUDASurfelReconstruction(1000, W, H, 80.0, 80.0, 48.0, 32.0)
    d = torch.full((H, W), 5000, dtype=torch.int32).to(torch.uint16).cuda()
    normals, radius = torch.zeros((H, W, 2), device="cuda"), torch.full((H, W), 1e-4, device="cuda")
    color = torch.zeros((H, W, 3), dtype=torch.uint8, device="cuda")
    rec.integrate(None, 0, IntegrateParams.defaults(), d, normals, radius, color, np.eye(4, dtype=np.float32)[:3])
    with pytest.raises(SurfelError) as e:
        rec.surfels_size()
    assert e.value.code == _lib.SM_ERR_CAPACITY


def test_invalid_arguments(product):
    with pytest.raises(SurfelError):
        R.CUDASurfelReconstruction(0, 64, 48, 50.0, 50.0, 32.0, 24.0)
    z = u16(48, 64)
    with pytest.raises(SurfelError):
        R.ErodeDepthMapCUDA(None, 4, z, u16(48, 64))
    with pytest.raises(SurfelError):
        R.OutlierDepthMapFusionCUDA(None, 0.02, z, 50.0, 50.0, 32.0, 24.0, [z, z, z], np.zeros((3, 12), np.float32),
                                    u16(48, 64))


FULL_SIZE_SIGMAS = [None, 0.01, 0.05]


def full_size_case(sigma):
    cam_ = S.Camera.tum(640, 480)
    st = S.make_stream(cam_, 40, stream_id=0, sigma_depth=sigma, device="cuda")
    return cam_, st, PreprocessParams.defaults(), IntegrateParams.defaults()


def stream_counts(s):
    """The counts of a free-running sm_stream_run that the tests compare with the reference's."""
    return {"frames_integrated": int(s.frames_integrated), "surfels_size": int(s.surfels_size),
            "surfel_count": int(s.surfel_count), "kernel_launches": int(s.kernel_launches)}


@pytest.mark.parametrize("sigma", FULL_SIZE_SIGMAS)
def test_full_size_stream_properties(product, sigma):
    """BASELINE configs 2 and 5 shapes (640x480; sigma_depth 0.05 m for the high-noise stream):
    free-running product vs. the free-running oracle's recorded counts over a stream; properties that
    do not depend on the reference's nondeterminism."""
    cam_, st, pp, ip = full_size_case(sigma)
    first, last = st.integrated_range()
    answers = oracle_answers()[f"full_size/{sigma}"]
    assert digest(st.depth.cpu().numpy()) == answers["inputs"], "the seeded input stream changed"
    sr = answers["stream"]
    rec_p = R.CUDASurfelReconstruction(2_000_000, 640, 480, cam_.fx, cam_.fy, cam_.cx, cam_.cy)
    sp = rec_p.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                          first, last)
    assert sp.frames_integrated == sr["frames_integrated"] == last - first
    # free-running counts drift (SURVEY §7): stay within 1 % of the oracle
    assert abs(int(sp.surfels_size) - sr["surfels_size"]) <= 0.01 * sr["surfels_size"]
    assert abs(int(sp.surfel_count) - sr["surfel_count"]) <= 0.01 * sr["surfel_count"]
    assert sp.kernel_launches < sr["kernel_launches"] / 2
    rows, n, merges = rec_p.dump_state()
    assert n == sp.surfels_size and n - merges == sp.surfel_count
    check_state_invariants(rows, n)
    if sigma == 0.05:
        # sigma_depth = 0.05 m is 2.5 % of a 2 m depth: the 2 % multi-frame outlier test (a2) rejects
        # (nearly) everything, in the product exactly as in the oracle
        assert sr["surfels_size"] < 2000
    else:
        assert n > 50_000
    if n:
        stamps = rows[17].view(np.uint32)
        assert stamps.min() >= first and stamps.max() < last, "creation stamps are frame indices of the stream"
    # host-resident (pinned) frames give the same result as device-resident frames
    rec_h = R.CUDASurfelReconstruction(2_000_000, 640, 480, cam_.fx, cam_.fy, cam_.cx, cam_.cy)
    sh = rec_h.stream_run(None, st.depth.cpu().pin_memory(), st.color.cpu().pin_memory(), st.global_T_frame,
                          st.frame_T_global, st.others_TR_reference, pp, ip, first, last)
    assert sh.h2d_bytes > 0
    assert abs(int(sh.surfels_size) - int(sp.surfels_size)) <= 0.002 * sp.surfels_size + 5
    # sm_stream_run overlaps the kernels of three frames in its frame graph; with stage timings
    # enabled it runs them one after the other on the caller's stream. Same result either way
    # (up to the float-atomic rounding that also separates two runs of the reference).
    rec_s = R.CUDASurfelReconstruction(2_000_000, 640, 480, cam_.fx, cam_.fy, cam_.cx, cam_.cy)
    rec_s.enable_timings(True)
    ss = rec_s.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                          first, last)
    assert abs(int(ss.surfels_size) - int(sp.surfels_size)) <= 0.002 * sp.surfels_size + 5
    assert abs(int(ss.surfel_count) - int(sp.surfel_count)) <= 0.002 * sp.surfel_count + 5
    assert len(rec_s.GetTimings()) == 7


def test_device_timeline_of_the_frame_graph(product):
    """sm_timeline_enable: the kernels stamp their own start / end while sm_stream_run overlaps three
    frames in its frame graph. The stamps must respect the data dependencies of the frame DAG
    (DESIGN.md): associate after project, integrate after blend and merge, regularisation after
    the neighbour update and the creation, the next frame's integration after this frame's
    regularisation, the next frame's projection after this frame's creation."""
    import ctypes as C
    cam_ = S.Camera.tum(320, 240)
    st = S.make_stream(cam_, 24, stream_id=1, device="cuda")
    pp, ip = PreprocessParams.defaults(), IntegrateParams.defaults()
    first, last = st.integrated_range()
    rec = R.CUDASurfelReconstruction(500_000, 320, 240, cam_.fx, cam_.fy, cam_.cx, cam_.cy)
    frames = 32
    product.call("timeline_enable", rec._h, frames)
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    kernels = product.fn["profile_kernel_count"]()
    names = [product.fn["profile_kernel_name"](i).decode() for i in range(kernels)]
    buf = np.zeros((frames, kernels, 2), dtype=np.uint64)
    product.call("timeline_read", rec._h, buf.ctypes.data_as(C.POINTER(C.c_uint64)), frames)
    product.call("timeline_enable", rec._h, 0)
    k = {n: i for i, n in enumerate(names)}
    never = np.uint64(0xFFFFFFFFFFFFFFFF)

    def start(f, name):
        return int(buf[f, k[name], 0])

    def end(f, name):
        return int(buf[f, k[name], 1])

    chain = ["k_project", "k_associate", "k_blend", "k_integrate", "k_update_neighbors", "k_reg_accumulate",
             "k_reg_step"]
    for f in range(first + 2, last):
        for name in chain + ["k_merge", "k_new_surfel_scan", "k_create_surfels", "k_bilateral_outlier",
                             "k_erode_normals_radii"]:
            assert buf[f, k[name], 0] != never, (f, name)
            assert end(f, name) >= start(f, name)
        for a, b in zip(chain[:-1], chain[1:]):
            assert start(f, b) >= end(f, a), (f, a, b)
        assert start(f, "k_merge") >= end(f, "k_associate")
        assert start(f, "k_integrate") >= end(f, "k_merge")
        assert start(f, "k_new_surfel_scan") >= end(f, "k_blend")
        assert start(f, "k_create_surfels") >= max(end(f, "k_new_surfel_scan"), end(f, "k_integrate"))
        assert start(f, "k_reg_accumulate") >= end(f, "k_create_surfels")
        assert start(f, "k_project") >= end(f, "k_erode_normals_radii")
        if f + 1 < last:
            assert start(f + 1, "k_integrate") >= end(f, "k_reg_step")
            assert start(f + 1, "k_project") >= end(f, "k_integrate")
            assert start(f + 1, "k_project") >= end(f, "k_create_surfels")


LARGE_FRAME_FIRST_ROWS = (0, 1, 2, 7, 8, 9, 10, 17, 18, 24)


def large_frame_case():
    width, height = 1280, 960
    cam_ = S.Camera(width, height, 1050.0, 1050.0, 640.0, 480.0)
    st = S.make_stream(cam_, 16, stream_id=2, device="cuda")
    pp, ip = PreprocessParams.defaults(), IntegrateParams.defaults()
    pp.depth_valid_region_radius = cam_.valid_region_radius()
    return cam_, st, pp, ip, 20_000_000


def first_frame_row_digests(rows, n):
    return {str(row): digest(rows[row, :n].view(np.uint32)) for row in LARGE_FRAME_FIRST_ROWS}


def test_large_frame_stream_properties(product):
    """BASELINE config 2 shape (1280x960 frames, 20 M surfel cap), shortened to 16 frames: the
    free-running product against the free-running oracle's recorded counts through size-independent
    properties, plus the exact quantities that do not depend on the reference's races (first frame: no
    surfels yet, so every pixel with a measurement creates exactly one surfel in both)."""
    cam_, st, pp, ip, cap = large_frame_case()
    first, last = st.integrated_range()
    answers = oracle_answers()["large_frame"]
    assert digest(st.depth.cpu().numpy()) == answers["inputs"], "the seeded input stream changed"
    rec_p = R.CUDASurfelReconstruction(cap, cam_.width, cam_.height, cam_.fx, cam_.fy, cam_.cx, cam_.cy)
    # first integrated frame only: deterministic in the reference as well
    sp1 = rec_p.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                           first, first + 1)
    assert sp1.surfels_size == answers["first_frame"]["surfels_size"] > 50_000
    rows_p, n_p, _ = rec_p.dump_state()
    got = first_frame_row_digests(rows_p, n_p)
    assert [row for row in got if got[row] != answers["first_frame"]["rows"][row]] == [], "rows differing from the reference"
    # whole stream
    rec_p.reset()
    sp = rec_p.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                          first, last)
    sr = answers["stream"]
    assert sp.frames_integrated == sr["frames_integrated"] == last - first
    assert abs(int(sp.surfels_size) - sr["surfels_size"]) <= 0.01 * sr["surfels_size"]
    assert abs(int(sp.surfel_count) - sr["surfel_count"]) <= 0.01 * sr["surfel_count"]
    rows, n, merges = rec_p.dump_state()
    assert n == sp.surfels_size and n - merges == sp.surfel_count
    check_state_invariants(rows, n)
