"""The front half of Integrate() - min depth, association, conflicting surfel, measurement blending - held to its
sequential restatement (tests/integrate_walk.c: iw_associate, iw_blend): the recorded reference frames, constructed
states and blend frames that reach every branch, and every named mutation of the walk visible on clear pixels.

CPU only. The constructed cases are built here and imported by tests/test_association_walk_gpu.py."""
import numpy as np
import pytest

from tests import integrate_walk as IW
from tests.test_integrate_walk_host import FLIPPED, ODD, VGA, build_case, integrate_params
from tests.util import golden_camera, golden_params, load_golden

BLEND_RADII = (1, 2, 3, 12, 17, 18, 33, 34, 39)   # 17 -> 18 and 33 -> 34: k_blend's x-halo grows; 39: the largest it takes
SMALL = (20, 12, 18.0, 17.0, 10.3, 6.1)            # smaller than one k_blend tile (32 x 40) and than the halo
TILE_SHORT = (31, 39, 30.0, 31.0, 15.2, 19.7)
TILE = (32, 40, 30.0, 31.0, 16.1, 20.2)
TILE_PAST = (33, 41, 30.0, 31.0, 16.6, 20.4)
LARGE = (1280, 960, 1050.0, 1050.0, 639.5, 479.5)

# (name, camera, frame index, active window, surfels per pixel, blend radius, surfel count: None or the offset from a
# multiple of 1024)
CASES = [
    ("small-r3", SMALL, 5, 2, 3.0, 3, -1),
    ("tile-short-r12", TILE_SHORT, 1000, 2**31 - 1, 2.0, 12, 1),
    ("tile-r17", TILE, 5, 2, 2.0, 17, -1),
    ("tile-past-r18", TILE_PAST, 1000, 2, 2.0, 18, 1),
    ("odd-r2", ODD, 5, 2**31 - 1, 1.5, 2, None),
    ("odd-r33", ODD, 1000, 2, 1.5, 33, -1),
    ("flipped-r1", FLIPPED, 5, 2, 2.0, 1, 1),
    ("flipped-r34", FLIPPED, 1000, 2**31 - 1, 2.0, 34, None),
    ("vga-r39", VGA, 1000, 2**31 - 1, 1.6, 39, None),
    ("vga-r12", VGA, 5, 2, 1.2, 12, -1),
    ("large-r12", LARGE, 1000, 2**31 - 1, 0.5, 12, None),
]
HOST_CASES = [c for c in CASES if c[1] not in (VGA, LARGE)]


def _tile_crossing(extent, tile, fraction):
    """A position near `fraction` of the extent on a k_blend tile edge (a multiple of `tile`), where the extent has one."""
    return max(tile, int(round(fraction * extent / tile)) * tile) if extent > tile + 8 else int(fraction * extent)


def front_case(camera, frame_index, window, per_pixel, count_offset=None, seed=0):
    """build_case's state and frame, reworked for the front half: a clean supported region with holes that cross the
    k_blend tile edges (x = 32 k, y = 40 k), two holes whose rings meet, a hole on the image border, an unsupported
    region (its surfels have radius 0) with isolated supported pixels in it, and surfels at the edges of the
    projection: z just above 0, u = 0, u = W, v = 0, and z exactly at the occlusion depth. Returns (rows, frame, g32,
    l32)."""
    W, H, fx, fy, cx, cy = camera
    rows, frame, g32, l32 = build_case(camera, frame_index, window, per_pixel, seed)
    rng = np.random.default_rng(seed + 3 * W + H)
    depth = frame["depth_pre"].copy()
    yy, xx = np.mgrid[0:H, 0:W]
    plane = np.round(5000 * (1.0 + 0.0004 * (xx + 0.5) + 0.0003 * (yy + 0.5))).astype(np.uint16)
    clean = (xx < 0.5 * W) & (yy >= 0.05 * H) & (yy < 0.95 * H)
    depth[clean] = plane[clean]
    tx, ty = _tile_crossing(W, 32, 0.25), _tile_crossing(H, 40, 0.5)
    hw, hh = max(2, W // 16), max(2, H // 10)
    hole = (np.abs(xx - tx) < hw) & (np.abs(yy - ty) < hh)
    hole |= (np.abs(xx - (tx + 2 * hw + max(4, W // 20))) < max(1, hw // 2)) & (np.abs(yy - ty) < hh)   # a second front
    hole |= (xx < max(1, W // 40)) & (np.abs(yy - 0.75 * H) < hh)                                     # on the border column
    hole |= (yy < 1) & (np.abs(xx - 0.3 * W) < hw)                                                   # on the border row
    depth[hole] = 0
    frame = dict(frame, depth_pre=depth, depth=depth)
    # the unsupported region: the surfels that project into it keep their place but get radius 0
    local = l32[:, :3].astype(np.float64) @ rows[0:3].astype(np.float64) + l32[:, 3:].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = fx * local[0] / local[2] + cx, fy * local[1] / local[2] + cy
    ux0 = _tile_crossing(W, 32, 0.7) - W // 6
    unsupported = (u >= ux0) & (u < ux0 + W // 3) & (v >= 0.15 * H) & (v < 0.75 * H) & (rng.random(u.size) > 0.01)
    rows = rows.copy()
    rows[7, unsupported & (rows[7] > 0)] = 0.0
    # surfels at the edges of the projection, each a copy of a visible surfel moved in its camera frame
    n_edge = 48
    src = rng.choice(np.flatnonzero((local[2] > 0.5) & (rows[7] > 0)), n_edge)
    loc = local[:, src].copy()
    kind = np.arange(n_edge) % 6
    z = loc[2]
    loc[0, kind == 0] = (0.0 - cx) / fx * z[kind == 0]                        # u = 0
    loc[0, kind == 1] = (W - cx) / fx * z[kind == 1]                          # u = W
    loc[1, kind == 2] = (0.0 - cy) / fy * z[kind == 2]                        # v = 0
    tiny = kind == 3                                                          # z just above 0
    loc[:, tiny] *= np.float64(2.0 ** -60)
    edge = np.zeros((IW.ROW_COUNT, n_edge), np.float32)
    edge[:] = rows[:, src]
    g = g32.astype(np.float64)
    edge[0:3] = g[:, :3] @ loc + g[:, 3:]
    # z exactly at the occlusion depth (1 + sensor noise) * measurement: the surfel's own z decides `>` against `>=`
    at = (kind >= 4)
    e_local = l32[:, :3].astype(np.float64) @ edge[0:3].astype(np.float64) + l32[:, 3:].astype(np.float64)
    px = np.clip((fx * e_local[0] / e_local[2] + cx).astype(int), 0, W - 1)
    py = np.clip((fy * e_local[1] / e_local[2] + cy).astype(int), 0, H - 1)
    for j in np.flatnonzero(at):
        d = depth[py[j], px[j]]
        if d == 0:
            continue
        target = np.float32(np.float32(1.05) * (np.float32(d) * np.float32(1.0 / 5000.0)))
        scale = float(target) / e_local[2, j]
        edge[0:3, j] = (g[:, :3] @ (e_local[:, j] * scale) + g[:, 3])   # the transform rounds: some land on it
    rows = np.concatenate([rows, edge], axis=1)
    if count_offset is not None:
        n = rows.shape[1]
        target_n = (n // 1024) * 1024 + count_offset
        assert 0 < target_n and n - target_n < 2349   # only the merged tail of build_case is cut
        if target_n > n:
            rows = np.concatenate([rows, np.repeat(rows[:, -1:], target_n - n, axis=1)], axis=1)
        rows = rows[:, :target_n]
    return np.ascontiguousarray(rows), frame, g32, l32


def front_params(window, radius):
    ip = integrate_params(window, 1)
    ip.measurement_blending_radius = radius
    return ip


def blend_frame(W, H, seed):
    """A frame for the blend alone: depth, counts and sums built to reach every ring case at every radius: wide holes
    and wide unsupported regions (both rings run the full radius), fronts across the tile edges, isolated supported
    pixels, fronts that meet, ring pixels on the border rows and columns, counts 1 .. 9 (inexact reciprocals)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    depth = np.round(5000 * (1.0 + 0.0005 * xx + 0.0002 * yy + 0.01 * np.sin(xx / 7.0))).astype(np.uint16)
    supported = np.ones((H, W), bool)
    for _ in range(6):
        x0, y0 = rng.integers(0, W), rng.integers(0, H)
        w, h = rng.integers(2, max(3, W // 5)), rng.integers(2, max(3, H // 5))
        depth[y0:y0 + h, x0:x0 + w] = 0
    for _ in range(4):
        x0, y0 = rng.integers(0, W), rng.integers(0, H)
        w, h = rng.integers(4, max(5, W // 3)), rng.integers(4, max(5, H // 3))
        supported[y0:y0 + h, x0:x0 + w] = False
    supported |= rng.random((H, W)) < 0.01          # isolated supported pixels
    depth[rng.random((H, W)) < 0.002] = 0            # isolated holes
    depth[:, W // 2] = np.where(yy[:, 0] % 9 == 0, 0, depth[:, W // 2])
    if seed % 2:
        depth[0, :] = 0
        depth[:, -1] = 0
    if W >= 200:   # one hole and one unsupported band in clean surroundings: both rings run the largest radius out
        depth = np.where(depth == 0, 1, depth).astype(np.uint16)
        depth[50:60, 10:20] = 0
        supported = xx < 120
    counts = np.where(supported, rng.integers(1, 10, size=(H, W)), 0).astype(np.uint32)
    z = depth.astype(np.float64) / 5000.0
    per = z[..., None] * (1 + rng.normal(0, 0.004, size=(H, W, 9)))
    sums = np.zeros((H, W), np.float32)
    for k in range(9):   # float32 sums in index order: one legal summation order
        sums = np.where(k < counts, (sums + per[..., k].astype(np.float32)).astype(np.float32), sums)
    return depth, counts, sums


BLEND_FRAMES = [(W, H, seed) for seed, (W, H) in enumerate([(20, 12), (31, 39), (32, 40), (33, 41), (97, 83), (160, 120), (200, 110)])]


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def golden_association(g, f, mutations=()):
    cam = golden_camera(g)
    ip = golden_params(g)[1]
    before = g[f"f{f - 1}_state"] if f > int(g["frames"][0]) else np.zeros((IW.ROW_COUNT, 0), np.float32)
    return IW.associate(before, g[f"f{f}_pre_depth"], g[f"f{f}_normals"], cam, ip, f, g["frame_T_global"][f], mutations)


@pytest.mark.parametrize("f", [4, 5, 6, 7])
def test_association_matches_the_recorded_reference(golden, f):
    """From the recorded state of frame f - 1 and the recorded pre-blend depth and normals, the walk gives the
    reference's min depth, counts and conflicting surfels on clear pixels; the recorded winner is one of the walk's
    supporters and the recorded depth sums lie within the order bound."""
    res = golden_association(golden, f)
    rasters = {k[len(f"f{f}_"):]: v for k, v in golden.items() if k.startswith(f"f{f}_")}
    stats = IW.hold_association(res, rasters, winner="member", label=f"golden frame {f}")
    print(f"golden frame {f}: {stats}")
    assert stats["unclear"] <= 0.005 * stats["pixels"]


@pytest.mark.parametrize("f", [4, 5, 6, 7])
def test_blend_matches_the_recorded_reference(golden, f):
    """From the recorded counts and depth sums, the walk's blend gives the reference's blended depth bit for bit on
    every pixel whose range is one value, and inside the range elsewhere: no allowance for differing pixels."""
    ip = golden_params(golden)[1]
    res = IW.blend(golden[f"f{f}_pre_depth"], golden[f"f{f}_supporting_surfel_counts"],
                   golden[f"f{f}_supporting_surfel_depth_sums"], ip.measurement_blending_radius, ip.depth_scaling)
    stats = IW.hold_blend(res, golden[f"f{f}_blended_depth"], label=f"golden frame {f}")
    print(f"golden frame {f}: {stats}")
    assert res.branch["start_depth_zero"] == 0
    assert stats["ranged"] <= 0.005 * stats["pixels"]


@pytest.fixture(scope="module")
def host_fronts():
    out = []
    for name, camera, frame_index, window, per_pixel, radius, offset in HOST_CASES:
        ip = front_params(window, radius)
        rows, frame, g32, l32 = front_case(camera, frame_index, window, per_pixel, offset)
        args = (rows, frame["depth_pre"], frame["normals"], camera, ip, frame_index, l32)
        out.append((name, args, IW.associate(*args)))
    return out


@pytest.fixture(scope="module")
def host_blends(host_fronts):
    """(label, args, result) of the blend: the blend frames at every radius, and each constructed state's own
    association at its radius."""
    out = []
    for W, H, seed in BLEND_FRAMES:
        depth, counts, sums = blend_frame(W, H, seed)
        for radius in BLEND_RADII:
            args = (depth, counts, sums, radius, 5000.0)
            out.append((f"blend {W}x{H} r{radius}", args, IW.blend(*args)))
    for (name, a, res), case in zip(host_fronts, HOST_CASES):
        H, W = res.shape
        args = (a[1], res.counts.reshape(H, W), res.sum_float.reshape(H, W), case[5], 5000.0)
        out.append((name, args, IW.blend(*args)))
    return out


# Must be reached zero times: the argument that the start step's in-place depth write is harmless (iw_blend).
NEVER = {"start_depth_zero"}


def test_constructed_cases_reach_every_branch(host_fronts, host_blends):
    total = {b: 0 for b in IW.FRONT_BRANCHES}
    unclear = pixels = ranged = blend_pixels = 0
    for name, args, res in host_fronts:
        for b, v in res.branch.items():
            total[b] += v
        unclear += int(res.unclear.sum())
        pixels += res.first.size
    for name, args, res in host_blends:
        for b, v in res.branch.items():
            total[b] += v
        ranged += int((res.lo != res.hi).sum())
        blend_pixels += res.depth.size
    print("front-half branch counters over the host cases:", total)
    print(f"unclear association pixels: {unclear} of {pixels} ({100.0 * unclear / pixels:.3f} %); blended pixels with a "
          f"range: {ranged} of {blend_pixels} ({100.0 * ranged / blend_pixels:.3f} %)")
    for ring in (0, 1):   # each ring runs the largest radius to its end somewhere
        full = [name for name, args, res in host_blends if args[3] == 39 and res.level_counts[ring, 38] > 0]
        print(f"ring {ring} reaches level 38 of radius 39 in:", full)
        assert full
    missing = [b for b, v in total.items() if v < 5 and b not in NEVER]
    assert not missing, f"branches the constructed cases do not reach five times: {missing}"
    assert all(total[b] == 0 for b in NEVER)
    assert unclear <= 0.005 * pixels and ranged <= 0.005 * blend_pixels


def association_outputs(res):
    return (res.first.view(np.uint32), res.counts, IW.supporter_pairs(res), res.conflict_legal, res.conflict_any)


def changed_clear_pixels(base, other):
    """Clear pixels (in both walks) whose min depth, count, supporter set or legal conflicting set differ."""
    clear = ~(base.unclear | other.unclear)
    P = base.first.size
    differ = (base.first.view(np.uint32) != other.first.view(np.uint32)) | (base.counts != other.counts)
    for a, b in ((IW.supporter_pairs(base), IW.supporter_pairs(other)), (base.conflict_legal, other.conflict_legal)):
        sym = np.setxor1d(a, b)
        differ[(sym >> np.uint64(32)).astype(np.int64) % P] = True
    differ |= base.conflict_any != other.conflict_any
    return int((differ & clear).sum())


MUTATION_MINIMUM = 5


@pytest.mark.parametrize("mutation", IW.ASSOCIATION_MUTATIONS)
def test_every_association_mutation_changes_clear_pixels(host_fronts, mutation):
    changed = sum(changed_clear_pixels(res, IW.associate(*args, mutations=(mutation,))) for _, args, res in host_fronts)
    print(f"mutation {mutation}: {changed} clear pixels change on the constructed states")
    assert changed >= MUTATION_MINIMUM


@pytest.mark.parametrize("mutation", IW.BLEND_MUTATIONS)
def test_every_blend_mutation_changes_clear_pixels(host_blends, mutation):
    changed = 0
    for name, args, res in host_blends:
        other = IW.blend(*args, mutations=(mutation,))
        clear = (res.lo == res.hi) & (other.lo == other.hi)
        changed += int(((res.depth != other.depth) & clear).sum())
    print(f"mutation {mutation}: {changed} clear pixels change on the blend cases")
    assert changed >= MUTATION_MINIMUM
