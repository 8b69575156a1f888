"""The production pre-processing path (sm_preprocess: k_bilateral_outlier, then the TMA-filled k_erode_normals_radii)
on every parameter branch and at frame sizes around its tiles, checked three ways:
  (a) bit for bit against the stage API (sm_bilateral_filter_and_depth_cutoff ... sm_compute_point_radii...) on the
      same inputs: depth, normals, and radius where the normals stage kept the pixel;
  (b) the stage outputs against the float64 restatement of tests/preprocess_walk.py and the normals / radii anchors
      of tests/test_camera_geometry_gpu.py;
  (c) where the oracle is built (oracle/_ref), bit for bit against the reference library's own sm_preprocess.
"""
import itertools
from functools import lru_cache

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, SurfelError
from tests import preprocess_walk as P
from tests.test_camera_geometry_gpu import Unprojection, f32, normals64, radii64
from tests.test_parity_gpu import run_stages
from tests.test_session_gpu import assert_one_frame_equal
from tests.util import count_mismatch, other_frames

pytestmark = pytest.mark.gpu

CANARY_U16 = 0xBEEF
CANARY_F32 = -12345.0


def reference_or_none():
    return _lib.load_reference_oracle() if _lib.REF_LIB_PATH.exists() else None


def padded(shape, dtype, canary, pad):
    """A tensor of `shape` viewed out of a wider one whose extra columns hold `canary` (pad 0: contiguous)."""
    H, W = shape[:2]
    full = torch.full((H, W + pad) + tuple(shape[2:]), canary, dtype=dtype, device="cuda")
    return full, full[:, :W]


def run_fused(lib, cam, pp, raw, others, mats, pad=0):
    """rec.preprocess through `lib`: (depth, normals, radius) as numpy; with `pad` the outputs are pitched and
    their padding must come back untouched."""
    W, H, fx, fy, cx, cy = cam
    rec = R.CUDASurfelReconstruction(1024, W, H, fx, fy, cx, cy, lib=lib)
    bufs = [padded((H, W), torch.uint16, CANARY_U16, pad), padded((H, W, 2), torch.float32, CANARY_F32, pad),
            padded((H, W), torch.float32, CANARY_F32, pad)]
    rec.preprocess(None, pp, raw, others, mats, *[b[1] for b in bufs])
    torch.cuda.synchronize()
    rec.close()
    if pad:
        for full, _ in bufs:
            tail = full[:, W:].cpu().numpy()
            want = CANARY_U16 if full.dtype == torch.uint16 else CANARY_F32
            assert (tail == want).all(), "pitched output padding overwritten"
    return [b[1].cpu().numpy() for b in bufs]


def stage_outputs(cam, pp, raw, others, mats):
    o = run_stages(None, cam, pp, raw, others, mats)
    return {k: v.cpu().numpy() for k, v in o.items()}


def assert_fused_equals_stages(fused, st, label):
    d, n, r = fused
    assert count_mismatch(d, st["pre_depth"]) == 0, f"{label}: depth"
    assert count_mismatch(n, st["normals"]) == 0, f"{label}: normals"
    assert count_mismatch(r, st["radius"], st["normals_depth"] != 0) == 0, f"{label}: radius"


def assert_same_fused(a, b, written, label):
    assert count_mismatch(a[0], b[0]) == 0 and count_mismatch(a[1], b[1]) == 0, f"{label}: depth / normals"
    assert count_mismatch(a[2], b[2], written) == 0, f"{label}: radius"


class Walk:
    """Check (b) of one case; collects the worst fraction of every float64 bound used."""
    worst = {}

    @classmethod
    def note(cls, key, value):
        cls.worst[key] = max(cls.worst.get(key, 0.0), float(value))

    @classmethod
    def check(cls, camera, pp, raw, others, mats, st, label, bil=None):
        W, H = camera.width, camera.height
        cam = (W, H, camera.fx, camera.fy, camera.cx, camera.cy)
        raw = np.asarray(raw)
        if bil is None:
            bil = P.Bilateral(raw, pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor,
                              pp.bilateral_filter_radius_factor, int(f32(pp.depth_scaling) * f32(pp.max_depth)),
                              pp.depth_valid_region_radius)
        bad, frac, share = bil.check(st["bilateral"])
        assert bad == 0, f"{label}: {bad} bilateral pixels off the float64 restatement"
        cls.note("bilateral", frac)
        cls.note("bilateral margin share", share)
        out = P.Outlier(st["bilateral"], cam, others, mats, pp.outlier_filtering_depth_tolerance_factor,
                        pp.outlier_filtering_required_inliers)
        wrong, share = out.check(st["bilateral"], st["outlier"])
        assert wrong == 0, f"{label}: {wrong} outlier decisions off the float64 restatement"
        cls.note("outlier margin share", share)
        assert np.array_equal(P.erode64(st["outlier"], pp.depth_erosion_radius), st["erode"]), f"{label}: erosion"
        e, nd = st["erode"], st["normals_depth"]
        four = P.four_neighbours(e)
        assert not (nd != 0)[~four].any(), f"{label}: a pixel without its four neighbours kept by the normals stage"
        assert not st["normals"][~four].any(), f"{label}: a normal written without the four neighbours"
        U = Unprojection(camera, pp.depth_scaling)
        if H > 2 and W > 2:
            n64, keep64, valid, bound, dot_bound, dot = normals64(U, e, pp.observation_angle_threshold_deg)
            normals = st["normals"][1:-1, 1:-1].transpose(2, 0, 1).astype(np.float64)
            err = np.abs(normals - n64[:2]).max(axis=0)
            if valid.any():
                assert (err[valid] <= bound[valid]).all(), f"{label}: normal off by {(err / bound)[valid].max():.2f}x"
                with np.errstate(invalid="ignore", divide="ignore"):
                    cls.note("normal", np.nanmax(np.where(valid & (bound > 0), err / bound, 0.0)))
            threshold = -np.cos(np.pi / 180 * f32(pp.observation_angle_threshold_deg))
            clear = valid & (np.abs(dot - threshold) > dot_bound)
            assert count_mismatch(nd[1:-1, 1:-1] != 0, keep64, clear) == 0, f"{label}: normals keep / drop"
        assert np.array_equal(st["pre_depth"], np.where(P.neighbour_count(nd) >= 8, nd, 0)), f"{label}: isolated"
        r2, count, rel, _ = radii64(U, nd, f32(pp.point_radius_extension_factor), f32(pp.point_radius_clamp_factor))
        written = (nd != 0) & (count > 0)
        if written.any():
            with np.errstate(invalid="ignore", divide="ignore"):
                err = np.abs(st["radius"].astype(np.float64) - r2) / r2
            assert (err[written] <= rel[written]).all(), f"{label}: radius^2 off by {(err / rel)[written].max():.2f}x"
            cls.note("radius", (err / rel)[written].max())


@pytest.fixture(scope="module", autouse=True)
def report_bounds():
    yield
    if Walk.worst:
        print("\nworst fraction of each float64 bound used: " +
              ", ".join(f"{k} {v:.3f}" for k, v in sorted(Walk.worst.items())))


# ---------------------------------------------------------------------------------------
# parameter grid
# ---------------------------------------------------------------------------------------

FACTORS = {
    "erosion": [0, 1, 2, 3],
    "sigma_depth": [0.05, 0.1, 0.5],
    "sigma_xy": [3.0, 2.0, 1.0],
    "K": [2, 4, 6, 8],
    "required": ["all", "K-1", "1"],
    "clamp": [float("inf"), 1.2],
    "tail": ["default", "extension 1.0", "angle 60", "cutoffs"],
    "input": ["stream", "all zero", "unaligned raw", "pitched outputs"],
}


def pairwise_cover(factors):
    """Cases (dicts) in which every pair of levels of every two factors occurs at least once: each new case
    starts from the first uncovered pair and takes, factor by factor, the level that covers most new pairs."""
    names = list(factors)
    uncovered = {((a, i), (b, j)) for a, b in itertools.combinations(names, 2)
                 for i in range(len(factors[a])) for j in range(len(factors[b]))}
    cases = []
    while uncovered:
        (a, i), (b, j) = min(uncovered, key=lambda p: (names.index(p[0][0]), p[0][1], names.index(p[1][0]), p[1][1]))
        case = {a: i, b: j}
        for n in names:
            if n in case:
                continue
            def gain(level):
                trial = dict(case, **{n: level})
                return sum(((x, trial[x]), (y, trial[y])) in uncovered
                           for x, y in itertools.combinations(names, 2) if x in trial and y in trial)
            case[n] = max(range(len(factors[n])), key=lambda level: (gain(level), -level))
        uncovered -= {((x, case[x]), (y, case[y])) for x, y in itertools.combinations(names, 2)}
        cases.append({n: factors[n][case[n]] for n in names})
    return cases


GRID = pairwise_cover(FACTORS)
GRID_CAMERA = S.Camera.tum(160, 120)
FRAME = 4


@lru_cache(maxsize=None)
def grid_stream():
    return S.make_stream(GRID_CAMERA, 9, stream_id=41, device="cuda")


def grid_case(case):
    st = grid_stream()
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = GRID_CAMERA.valid_region_radius()
    pp.depth_erosion_radius = case["erosion"]
    pp.bilateral_filter_sigma_depth_factor = case["sigma_depth"]
    pp.bilateral_filter_sigma_xy = case["sigma_xy"]
    K = case["K"]
    pp.outlier_filtering_frame_count = K
    pp.outlier_filtering_required_inliers = {"all": -1, "K-1": K - 1, "1": 1}[case["required"]]
    pp.point_radius_clamp_factor = case["clamp"]
    if case["tail"] == "extension 1.0":
        pp.point_radius_extension_factor = 1.0
    elif case["tail"] == "angle 60":
        pp.observation_angle_threshold_deg = 60.0
    elif case["tail"] == "cutoffs":
        pp.max_depth = 1.75   # 8750 depth units in fp32 and in float64 alike
        pp.depth_valid_region_radius = 60.0
    raw = st.depth[FRAME]
    if case["input"] == "all zero":
        raw = torch.zeros_like(raw)
    elif case["input"] == "unaligned raw":
        wide = torch.zeros((GRID_CAMERA.height, GRID_CAMERA.width + 3), dtype=torch.uint16, device="cuda")
        wide[:, 1:GRID_CAMERA.width + 1] = raw
        raw = wide[:, 1:GRID_CAMERA.width + 1]
        assert raw.data_ptr() % 16 != 0 and (raw.stride(0) * 2) % 16 != 0
    others = [st.depth[f] for f in other_frames(FRAME, K)]
    mats = S.others_TR_reference(st.global_T_frame.astype(np.float64), pp.depth_scaling, K)[FRAME]
    return pp, raw, others, mats, (8 if case["input"] == "pitched outputs" else 0)


def test_grid_is_a_pairwise_cover():
    for a, b in itertools.combinations(FACTORS, 2):
        seen = {(c[a], c[b]) for c in GRID}
        assert len(seen) == len(FACTORS[a]) * len(FACTORS[b]), (a, b)
    assert len(GRID) < 30


@pytest.mark.parametrize("case", GRID, ids=lambda c: "-".join(f"{v}" for v in c.values()).replace(" ", "_"))
def test_fused_preprocess_parameter_grid(product, case):
    pp, raw, others, mats, pad = grid_case(case)
    cam = (GRID_CAMERA.width, GRID_CAMERA.height, GRID_CAMERA.fx, GRID_CAMERA.fy, GRID_CAMERA.cx, GRID_CAMERA.cy)
    # each case lands on the instantiation it names: radius 6 fused, 4 and 2 generic; the ignored-tap test dropped
    # exactly below sigma_depth 0.0675
    assert P.bilateral_radius(pp.bilateral_filter_sigma_xy, pp.bilateral_filter_radius_factor) == \
        {3.0: 6, 2.0: 4, 1.0: 2}[case["sigma_xy"]]
    assert P.ignored_taps_vanish(pp.bilateral_filter_sigma_depth_factor) == (case["sigma_depth"] < 0.0675)
    fused = run_fused(None, cam, pp, raw, others, mats, pad)
    st = stage_outputs(cam, pp, raw, others, mats)
    assert_fused_equals_stages(fused, st, "fused vs stages")
    others_np = [o.cpu().numpy() for o in others]
    Walk.check(GRID_CAMERA, pp, raw.cpu().numpy(), others_np, mats, st, str(case))
    if case["input"] == "all zero":
        assert not fused[0].any()
    else:
        assert fused[0].any(), "the case keeps pixels"
    ref = reference_or_none()
    if ref is not None:
        assert_same_fused(fused, run_fused(ref, cam, pp, raw, others, mats, pad), st["normals_depth"] != 0, "oracle")


@pytest.mark.parametrize("kind", ["tolerance", "required"])
def test_fused_outlier_decisions_on_designed_frames(product, kind):
    """Other frames built to put decisions where a wrong tolerance or inlier count shows: identity motions and
    depth ratios sweeping 0.96 - 1.04 across the columns (K = 2, all required), or three agreeing frames and a
    fourth 5 % off in the top half and a third 5 % off in the left half (K = 4, 3 required)."""
    cam = GRID_CAMERA
    W, H = cam.width, cam.height
    y, x = np.mgrid[0:H, 0:W]
    raw = (10000 + 2 * x + y).astype(np.uint16)
    pp = size_params(cam, 2)
    if kind == "tolerance":
        K, others = 2, [np.round(raw * (0.96 + 0.08 * x / (W - 1))).astype(np.uint16)] * 2
    else:
        K = 4
        off = np.where(y < H // 2, np.round(raw * 1.05), raw).astype(np.uint16)
        left = np.where(x < W // 2, np.round(raw * 0.95), raw).astype(np.uint16)
        others = [raw, raw, left, off]   # four agree bottom right, two top left, three elsewhere
        pp.outlier_filtering_required_inliers = 3
    pp.outlier_filtering_frame_count = K
    mats = np.zeros((K, 3, 4), np.float32)
    mats[:, :, :3] = np.eye(3)
    dev = lambda a: torch.from_numpy(a.astype(np.int32)).to(torch.uint16).cuda()
    camt = (W, H, cam.fx, cam.fy, cam.cx, cam.cy)
    raw_t, others_t = dev(raw), [dev(o) for o in others]
    fused = run_fused(None, camt, pp, raw_t, others_t, mats)
    st = stage_outputs(camt, pp, raw_t, others_t, mats)
    assert_fused_equals_stages(fused, st, kind)
    Walk.check(cam, pp, raw, others, mats, st, kind)
    kept = st["outlier"] != 0
    assert kept.any() and (~kept & (st["bilateral"] != 0)).any(), "both decisions occur"
    ref = reference_or_none()
    if ref is not None:
        assert_same_fused(fused, run_fused(ref, camt, pp, raw_t, others_t, mats), st["normals_depth"] != 0, "oracle")


# ---------------------------------------------------------------------------------------
# frame sizes around the tiles
# ---------------------------------------------------------------------------------------

SIZES = [(1, 1), (7, 3), (16, 8), (31, 15), (32, 16), (33, 17), (47, 25), (48, 26), (49, 27), (65, 33), (97, 41),
         (333, 201), (848, 480), (1280, 720)]
TILE_W, TAIL_TILE_H, HALO_Y, HALO_X, MAX_ERODE, BIL_TILE_H, BIL_R, BIL_PADX = 32, 16, 5, 8, 3, 4, 6, 8


def tail_index_ranges(width, height, r):
    """k_erode_normals_radii's shared-memory and global indices for every block and thread, restated: returns the
    (lowest, highest) index of each shared array next to its size, and asserts the guarded writes stay inside."""
    BW, BH = TILE_W + 2 * HALO_X, TAIL_TILE_H + 2 * HALO_Y
    EW, EH = TILE_W + 4, TAIL_TILE_H + 4
    HVH, NW, NH = EH + 2 * MAX_ERODE, TILE_W + 2, TAIL_TILE_H + 2
    ranges = {}

    def span(name, idx, size):
        lo, hi = int(np.min(idx)), int(np.max(idx))
        if name in ranges:
            lo, hi = min(lo, ranges[name][0]), max(hi, ranges[name][1])
        ranges[name] = (lo, hi, size)

    if r > 0:
        i = np.arange((EH + 2 * r) * EW)
        hy, ex = i // EW, i % EW
        base = (hy - r + HALO_Y - 2) * BW + ex + HALO_X - 2
        span("sB (row validity)", np.concatenate([base - r, base + r]), BH * BW)
        span("sHV (write)", i, HVH * EW)
    i = np.arange(EW * EH)
    ey, ex = i // EW, i % EW
    span("sB (erosion centre)", (ey + HALO_Y - 2) * BW + ex + HALO_X - 2, BH * BW)
    if r > 0:
        span("sHV (read)", np.concatenate([ey * EW + ex, (ey + 2 * r) * EW + ex]), HVH * EW)
    span("sE (write)", i, EH * EW)
    i = np.arange(NW * NH)
    ly, lx = i // NW, i % NW
    e = (ly + 1) * EW + lx + 1
    span("sE (normals)", np.concatenate([e - EW, e - 1, e + 1, e + EW]), EH * EW)
    span("sN (write)", i, NH * NW)
    t = np.arange(256)
    for half in range(TAIL_TILE_H // 8):
        lx, ly = t & 31, (t >> 5) + 8 * half
        span("sN (radii)", np.concatenate([(ly + 1 + dy) * NW + lx + 1 + dx for dy in (-1, 0, 1) for dx in (-1, 0, 1)]),
             NH * NW)
    for name, (lo, hi, size) in ranges.items():
        assert 0 <= lo and hi < size, (width, height, r, name, lo, hi, size)
    # guarded global writes of every block: normals on the interior of the N tile, radii / depth on the output tile
    gx_t, gy_t = np.meshgrid(np.arange(0, width + TILE_W - 1, TILE_W)[: (width + TILE_W - 1) // TILE_W],
                             np.arange(0, height + TAIL_TILE_H - 1, TAIL_TILE_H)[: (height + TAIL_TILE_H - 1) // TAIL_TILE_H])
    ly, lx = np.mgrid[1:TAIL_TILE_H + 1, 1:TILE_W + 1]
    gx = gx_t.reshape(-1, 1, 1) - 1 + lx
    gy = gy_t.reshape(-1, 1, 1) - 1 + ly
    guarded = (gx < width) & (gy < height)
    assert (gx[guarded] >= 0).all() and (gy[guarded] >= 0).all()
    assert ((gy * width + gx)[guarded] < width * height).all()
    # the fused bilateral kernel's tile fill: aligned 8-pixel loads only inside the row, the tile in shared memory
    SW, rows = TILE_W + 2 * BIL_PADX, BIL_TILE_H + 2 * BIL_R
    v = np.arange(rows * (SW // 8))
    row, col = v // (SW // 8), (v % (SW // 8)) * 8
    assert (row * SW + col + 7 < rows * SW).all()
    return ranges


@lru_cache(maxsize=None)
def size_inputs(width, height):
    """(camera, raw, others, mats [8, 3, 4], stage-independent bilateral walk) of one frame size: hand-built depth
    below 100 pixels of width, a synthetic stream above."""
    if width < 100:
        cam = S.Camera(width, height, 0.8 * max(width, 8), 0.8 * max(width, 8), width / 2.0, height / 2.0)
        y, x = np.mgrid[0:height, 0:width]
        d = 8000 + 3 * x + 2 * y
        d[:, width // 2:] += 400                      # a step
        d[(x == width // 3) & (y == height // 2)] = 0  # holes
        d[(x == (2 * width) // 3) & (y == height // 3)] = 0
        if width >= 8 and height >= 8:
            d[0, :] = d[-1, :] = d[:, 0] = d[:, -1] = 0  # zeros along every border
        raw = d.astype(np.uint16)
        others = [raw] * 8
        mats = np.zeros((8, 3, 4), np.float32)
        mats[:, :, :3] = np.eye(3)
        for k in range(8):   # small known motions: a fraction of a pixel sideways, a few depth units along z
            mats[k, :, 3] = ((-1) ** k * 0.3, (k % 3 - 1) * 0.2, (k - 3.5))
        raw_t = torch.from_numpy(raw.astype(np.int32)).to(torch.uint16).cuda()
        others_t = [raw_t] * 8
    else:
        cam = S.Camera(width, height, 525.0 * width / 640, 525.0 * width / 640, width / 2.0, height / 2.0)
        st = S.make_stream(cam, 9, stream_id=43, device="cuda")
        raw_t = st.depth[FRAME]
        others_t = [st.depth[f] for f in other_frames(FRAME, 8)]
        mats = st.others_TR_reference[FRAME]
    pp = size_params(cam, 2)
    bil = P.Bilateral(raw_t.cpu().numpy(), pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor,
                      pp.bilateral_filter_radius_factor, int(f32(pp.depth_scaling) * f32(pp.max_depth)),
                      pp.depth_valid_region_radius)
    return cam, raw_t, others_t, mats, bil


def size_params(cam, erosion):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    pp.depth_erosion_radius = erosion
    return pp


def test_tail_indices_stay_in_range_at_every_size():
    for (w, h), r in itertools.product(SIZES, range(MAX_ERODE + 1)):
        tail_index_ranges(w, h, r)


ACCEPTED = {}


@pytest.mark.parametrize("erosion", [2, 0, 3])
@pytest.mark.parametrize("width,height", SIZES)
def test_fused_preprocess_frame_sizes(product, width, height, erosion):
    tail_index_ranges(width, height, erosion)
    cam, raw, others, mats, bil = size_inputs(width, height)
    camt = (width, height, cam.fx, cam.fy, cam.cx, cam.cy)
    pp = size_params(cam, erosion)
    try:
        fused = run_fused(None, camt, pp, raw, others, mats)
    except SurfelError as e:
        assert e.code == _lib.SM_ERR_INVALID_ARGUMENT, f"sm_create at {width} x {height}: {e}"
        ACCEPTED[(width, height)] = False
        pytest.skip(f"sm_create refuses {width} x {height}: {e}")
    ACCEPTED[(width, height)] = True
    st = stage_outputs(camt, pp, raw, others, mats)
    assert_fused_equals_stages(fused, st, f"{width}x{height}")
    Walk.check(cam, pp, raw.cpu().numpy(), [o.cpu().numpy() for o in others], mats, st, f"{width}x{height}", bil)
    if min(width, height) >= 16 and (erosion < 3 or height > 16):   # radius 3 erodes 32 x 16 to nothing
        assert fused[0].any(), "the frame keeps pixels"
    ref = reference_or_none()
    if ref is not None:
        assert_same_fused(fused, run_fused(ref, camt, pp, raw, others, mats), st["normals_depth"] != 0, "oracle")


def test_report_accepted_sizes():
    if ACCEPTED:
        print("\nsm_create accepts: " + ", ".join(f"{w}x{h}" for (w, h), ok in ACCEPTED.items() if ok) +
              "; refuses: " + (", ".join(f"{w}x{h}" for (w, h), ok in ACCEPTED.items() if not ok) or "none"))


# ---------------------------------------------------------------------------------------
# the frame graph
# ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("erosion", [0, 3])
def test_frame_graph_and_session_preprocess_like_sm_preprocess(product, erosion):
    """sigma_depth 0.5 (the instantiation that keeps the ignored-tap test), K = 4 with 3 required: the first frame a
    9-frame sm_stream_run and a session integrate equals sm_preprocess + sm_integrate of that frame."""
    cam = S.Camera.tum(320, 240)
    st = S.make_stream(cam, 9, stream_id=47, device="cuda")
    pp = size_params(cam, erosion)
    pp.bilateral_filter_sigma_depth_factor = 0.5
    pp.outlier_filtering_frame_count, pp.outlier_filtering_required_inliers = 4, 3
    ip = IntegrateParams.defaults()
    K = 4
    others = R.stream_outlier_filter_transforms(st.global_T_frame, st.frame_T_global, K, st.depth_scaling)
    make = lambda: R.CUDASurfelReconstruction(400_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    direct, graph, session = make(), make(), make()
    H, W = cam.height, cam.width
    d = torch.zeros((H, W), dtype=torch.uint16, device="cuda")
    n, r = torch.zeros((H, W, 2), device="cuda"), torch.zeros((H, W), device="cuda")
    direct.preprocess(None, pp, st.depth[FRAME], [st.depth[f] for f in other_frames(FRAME, K)], others[FRAME], d, n, r)
    direct.integrate(None, FRAME, ip, d, n, r, st.color[FRAME], st.global_T_frame[FRAME], st.frame_T_global[FRAME])
    torch.cuda.synchronize()
    stats = graph.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, others, pp, ip, FRAME,
                             FRAME + 1)
    assert stats.frames_integrated == 1
    with session.session(pp, ip, (W, H), first_frame_index=FRAME - K // 2) as s:
        for f in range(FRAME - K // 2, FRAME + K // 2 + 1):
            s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
    assert s.stats.frames_integrated == 1
    assert_one_frame_equal(graph, direct)
    assert_one_frame_equal(session, direct)
