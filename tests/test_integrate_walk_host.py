"""The integration walk (tests/integrate_walk.c) held to the recorded reference, and the constructed states the GPU
test runs: every branch of the cycle reached, every named mutation of the walk visible on clear slots.

CPU only. The states are built here and imported by tests/test_integrate_walk_gpu.py."""
import numpy as np
import pytest

from oracle import cpu_walk
from surfelmeshing_b200._lib import IntegrateParams
from tests import integrate_walk as IW
from tests.util import golden_camera, golden_params, load_golden

COMPARED_ROWS = (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 17, 18, 19, 20, 21, 22, 24)

# (name, camera (W, H, fx, fy, cx, cy), frame index, active window, surfels per pixel, do_blending)
VGA = (640, 480, 525.0, 525.0, 319.5, 239.5)
ODD = (333, 201, 271.3, 263.9, 170.2, 97.6)
FLIPPED = (160, 120, 140.0, -138.0, 80.5, 59.5)   # negative fy
CASES = [
    ("odd-f5", ODD, 5, 2**31 - 1, 1.5, 0),
    ("odd-f1000-window2", ODD, 1000, 2, 1.5, 1),
    ("odd-fmax", ODD, 2**31 - 2, 2, 1.0, 1),
    ("flipped-f5-window2", FLIPPED, 5, 2, 2.0, 0),
    ("flipped-f1000", FLIPPED, 1000, 2**31 - 1, 2.0, 1),
    ("vga-f1000", VGA, 1000, 2**31 - 1, 1.6, 1),       # ~ 500 000 slots: beyond the resident grid of every kernel
]
HOST_CASES = [c for c in CASES if c[1] is not VGA]


def integrate_params(window, do_blending):
    ip = IntegrateParams.defaults()
    ip.surfel_integration_active_window_size = window
    ip.do_blending = do_blending
    # the cycle alone: no regularisation step, and a regularisation window that holds no slot, so the copy-only sweep
    # leaves the smooth positions as the cycle wrote them (its detach pass still runs, as in the walk)
    ip.regularization_iterations_per_integration_iteration = 0
    ip.regularization_frame_window_size = -1
    return ip


def build_case(camera, frame_index, window, per_pixel, seed=0):
    """A frame of hand-built rasters and a state that meets it in every way the cycle distinguishes. Returns
    (rows [25, n], frame dict, global_T_local, local_T_global)."""
    W, H, fx, fy, cx, cy = camera
    rng = np.random.default_rng(seed + W)
    a = 0.07
    G = np.array([[np.cos(a), 0, np.sin(a), 0.11], [0, 1, 0, -0.05], [-np.sin(a), 0, np.cos(a), 0.02]])
    g32 = G.astype(np.float32)
    l32 = IW.invert_rigid(g32)
    G = g32.astype(np.float64)

    def plane(u, v):
        return 1.0 + 0.0004 * u + 0.0003 * v

    # ---- the frame: a slanted plane; 8x8 blocks of holes, of far depth (surfels in front conflict) and of near depth
    # (surfels behind are occluded)
    yy, xx = np.mgrid[0:H, 0:W]
    block = rng.integers(0, 14, size=(H // 8 + 1, W // 8 + 1)).repeat(8, 0).repeat(8, 1)[:H, :W]
    z = plane(xx + 0.5, yy + 0.5) * np.select([block == 1, block == 2], [1.5, 0.8], 1.0)
    z = z * (1 + rng.choice([0.0, 0.0, 0.004, -0.004], size=z.shape))
    depth = np.round(5000 * z).astype(np.uint16)
    depth[block == 0] = 0
    depth[rng.random((H, W)) < 0.02] = 0
    normals = rng.normal(0, 0.04, size=(H, W, 2)).astype(np.float32)
    tilted = rng.random((H, W)) < 0.05
    normals[tilted, 0] = 0.75
    pixel_r2 = (1.2 * z / abs(fx)) ** 2
    radius = (pixel_r2 * rng.choice([1.0, 1.0, 1.0, 0.5, 3.0], size=z.shape)).astype(np.float32)
    color = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
    frame = dict(depth_pre=depth, depth=depth, normals=normals, radius=radius, color=color)

    # ---- the state, in raster order of the pixel a slot projects to (so slot i +- 1 and i +- a row are near)
    n = int(per_pixel * W * H)
    u = rng.uniform(-3, W + 3, n)
    v = rng.uniform(-3, H + 3, n)
    # a column of surfels in pixel column 1 and along the borders: the secondary-pixel rule's `px > 1`
    edge = rng.random(n) < 0.03
    u[edge] = rng.uniform(0, 2.2, edge.sum())
    order = np.argsort(np.floor(v) * (W + 8) + u, kind="stable")
    u, v = u[order], v[order]
    zs = plane(u, v) * (1 + rng.choice([0.002, -0.002, 0.011, -0.011, 0.0, 0.03, -0.03], size=n))
    local = np.stack([(u - cx) / fx * zs, (v - cy) / fy * zs, zs])
    r2 = (1.2 * zs / abs(fx)) ** 2 * rng.choice([1.0, 1.0, 1.0, 1.0, 0.3, 4.0], size=n)
    normal = np.tile(np.array([[0.0], [0.0], [-1.0]]), (1, n)) + rng.normal(0, 0.03, size=(3, n))
    kind = rng.random(n)
    tilt = kind < 0.08
    normal[:, tilt] = np.array([[0.0], [np.sin(0.9)], [-np.cos(0.9)]])
    normal[1, tilt] *= rng.choice([-1.0, 1.0], size=tilt.sum())            # two tilted neighbours can face apart: dot <= 0
    normal[:, (kind >= 0.08) & (kind < 0.11)] *= -1                       # back-facing
    normal /= np.linalg.norm(normal, axis=0)
    # near-copies of the previous slot: merge candidates on either side of each merge gate
    copy = np.flatnonzero(rng.random(n) < 0.18)
    copy = copy[copy > 0]
    for i in copy:   # in order, so a copy of a copy follows its original
        radius_factor = rng.choice([1.0, 1.0, 1.425, 1.455, 0.70, 0.689, 1.2])
        step = rng.choice([0.0, 0.0, 0.15, 0.35]) * np.sqrt(r2[i - 1])
        local[:, i] = local[:, i - 1] + np.array([step, 0.0, 0.0])
        r2[i] = r2[i - 1] * radius_factor
        if rng.random() < 0.15:   # a ratio of exactly 1.44f or 1 / 1.44f (float32), with an exact reciprocal: `>` against `>=`
            r2[i - 1] = 2.0 ** -16
            r2[i] = 2.0 ** -16 * rng.choice([1.4400000572204589844, 0.69444441795349121094])
        angle = rng.choice([0.0, 0.0, np.deg2rad(19.0), np.deg2rad(21.0)])
        c, s = np.cos(angle), np.sin(angle)
        nx, ny, nz = normal[:, i - 1]
        normal[:, i] = (nx, c * ny - s * nz, s * ny + c * nz)
    position = G[:, :3] @ local + G[:, 3:]
    gnormal = G[:, :3] @ normal

    rows = np.zeros((IW.ROW_COUNT, n), np.float32)
    ru = rows.view(np.uint32)
    rows[0:3] = position
    rows[3:6] = position + gnormal * rng.choice([0.0, 0.0, 0.0, 0.001, 0.05], size=n)   # smooth, some far from raw
    rows[6] = rng.choice([0.5, 1.0, 1.0, 2.0, 3.5, 4.5, 4.9, 5.0], size=n)
    rows[7] = r2
    rows[8:11] = gnormal
    ru[17] = np.where(rng.random(n) < 0.05, frame_index, 1)
    ru[18] = np.where(rng.random(n) < 0.2, frame_index - 3, frame_index - 1)
    ru[24] = rng.integers(0, 1 << 24, size=n, dtype=np.uint32) | (rng.random(n) < 0.1).astype(np.uint32) << 24
    special = rng.random(n)
    rows[7, special < 0.01] = 0.0                                        # radius 0: association skips it, merge does not
    gone = (special >= 0.01) & (special < 0.025)                         # merged in an earlier frame
    rows[7, gone] = -1.0
    ru[18, gone] = 0
    ru[24, gone] = (ru[24, gone] & 0xFFFFFF) | (1 << 24)
    row_step = max(int(per_pixel * (W + 6)), 2)
    offsets = rng.choice([-1, 1, 2, -2, -row_step, row_step, row_step + 1, 40 * row_step], size=(4, n))
    links = np.arange(n)[None, :] + offsets
    links = np.where((links < 0) | (links >= n) | (rng.random((4, n)) < 0.3), IW.INVALID, links)
    ru[19:23] = links.astype(np.uint32)

    # ---- whole segments behind the camera and whole segments of merged slots; a slot count off the 1024 grid
    def tail(count, behind):
        t = np.zeros((IW.ROW_COUNT, count), np.float32)
        tu = t.view(np.uint32)
        loc = np.stack([rng.uniform(-0.3, 0.3, count), rng.uniform(-0.2, 0.2, count),
                        np.full(count, -1.0 if behind else 1.05)])
        t[0:3] = G[:, :3] @ loc + G[:, 3:]
        t[3:6] = t[0:3]
        t[6] = 1.0
        t[7] = 1e-5 if behind else -1.0
        t[8:11] = (G[:, :3] @ np.array([[0.0], [0.0], [-1.0]]))
        tu[17] = 1
        tu[18] = frame_index - 1 if behind else 0
        tu[19:23] = IW.INVALID
        tu[24] = 0x808080 | (0 if behind else 1 << 24)
        return t
    rows = np.concatenate([rows, tail(2048 + 512, True), tail(2048 + 301, False)], axis=1)
    assert rows.shape[1] % 1024 != 0
    return np.ascontiguousarray(rows), frame, g32, l32


def host_rasters(rows, frame, camera, ip, frame_index, l32):
    """One legal outcome of the association, from the plain-C walk of the reference's association kernel."""
    W, H, fx, fy, cx, cy = camera
    return cpu_walk.associate(rows, frame_index, fx, fy, cx, cy, l32, frame["depth_pre"], frame["normals"],
                              ip.sensor_noise_factor, ip.normal_compatibility_threshold_deg, ip.depth_scaling,
                              ip.surfel_integration_active_window_size)


def changed_clear_slots(base, other):
    """Clear slots (in both walks) whose compared rows differ."""
    n = min(base.n_after, other.n_after)
    differ = np.any(base.rows[list(COMPARED_ROWS), :n].view(np.uint32) != other.rows[list(COMPARED_ROWS), :n].view(np.uint32), axis=0)
    clear = ((base.status[:n] | other.status[:n]) & (IW.ST_UNCLEAR | IW.ST_LINKS_UNCLEAR)) == 0
    return int((differ & clear).sum()) + abs(base.n_after - other.n_after)


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def golden_walk(g, f, mutations=()):
    first = int(g["frames"][0])
    before = g[f"f{f - 1}_state"] if f > first else np.zeros((IW.ROW_COUNT, 0), np.float32)
    frame = dict(depth_pre=g[f"f{f}_pre_depth"], depth=g[f"f{f}_blended_depth"], normals=g[f"f{f}_normals"],
                 radius=g[f"f{f}_radius"], color=g["color"][f])
    rasters = {k[len(f"f{f}_"):]: v for k, v in g.items() if k.startswith(f"f{f}_")}
    res = IW.walk(before, frame, rasters, golden_camera(g), golden_params(g)[1], f, g["global_T_frame"][f],
                  g["frame_T_global"][f], mutations)
    return before, rasters, res


@pytest.mark.parametrize("f", [4, 5, 6, 7])
def test_walk_matches_the_recorded_reference(golden, f):
    """The walk, fed with the REFERENCE's recorded rasters, the recorded state of frame f - 1 and the recorded blended
    depth, gives the recorded state of frame f: flags, rows, links, new-surfel rasters and counters. The recording
    ran the regulariser too, which moves smooth positions (not compared here) and drops links; slots whose merge
    partner merged in the same frame are excused (the reference merges in place)."""
    before, rasters, res = golden_walk(golden, f)
    chain = (res.status & IW.ST_MERGE_CHAIN) != 0
    stats = IW.hold(res, before, golden[f"f{f}_state"], rasters["new_surfel_flag_vector"], rasters["new_surfel_indices"],
                    excused=chain, smooth=False, links_may_drop=True, label=f"golden frame {f}")
    n, merges = [int(v) for v in golden[f"f{f}_counts"]]
    merges_before = int(golden[f"f{f - 1}_counts"][1]) if f > int(golden["frames"][0]) else 0
    print(f"golden frame {f}: {stats}, merges {res.merges} (recorded {merges - merges_before})")
    assert n == res.n_after
    assert abs((merges - merges_before) - res.merges) <= res.unclear_merges + stats["excused"]
    assert stats["unclear"] <= 0.002 * stats["slots"] and stats["links_unclear"] <= 0.06 * stats["slots"]
    assert stats["links_dropped"] <= 0.02 * stats["slots"]


# Branches every constructed case set must reach, with the least count over all host cases together.
UNREACHED_BY_CONSTRUCTION = {
    # the partner of a merging slot is its pixel's winner, and a winner passed `radius^2 > 0` in the association
    "merge_partner_merged",
    # a surfel wins at most its primary and its secondary pixel, which are 4-adjacent: never two of the four pixels
    # around a third one
    "nu_same_twice",
    # the partner is the pixel's winner; it merges itself only where it lost its own primary pixel (counted, not required)
    "merge_chain",
}


@pytest.fixture(scope="module")
def host_walks():
    out = []
    for name, camera, frame_index, window, per_pixel, blending in HOST_CASES:
        ip = integrate_params(window, blending)
        rows, frame, g32, l32 = build_case(camera, frame_index, window, per_pixel)
        rasters = host_rasters(rows, frame, camera, ip, frame_index, l32)
        args = (rows, frame, rasters, camera, ip, frame_index, g32, l32)
        out.append((name, args, IW.walk(*args)))
    return out


def test_constructed_states_reach_every_branch(host_walks):
    total = {b: 0 for b in IW.BRANCHES}
    unclear = links_unclear = slots = 0
    for name, args, res in host_walks:
        for b, v in res.branch.items():
            total[b] += v
        unclear += int(((res.status & IW.ST_UNCLEAR) != 0).sum())
        links_unclear += int(((res.status & (IW.ST_UNCLEAR | IW.ST_LINKS_UNCLEAR)) == IW.ST_LINKS_UNCLEAR).sum())
        slots += res.n_after
    print("branch counters over the host cases:", total)
    print(f"unclear slots: {unclear} of {slots} ({100.0 * unclear / slots:.3f} %); clear but for their links: "
          f"{links_unclear} ({100.0 * links_unclear / slots:.3f} %)")
    missing = [b for b, v in total.items() if v < 5 and b not in UNREACHED_BY_CONSTRUCTION]
    assert not missing, f"branches the constructed states do not reach five times: {missing}"
    assert unclear <= 0.005 * slots and links_unclear <= 0.08 * slots


MUTATION_MINIMUM = 5


@pytest.mark.parametrize("mutation", sorted(IW.MUTATIONS))
def test_every_mutation_changes_clear_slots(host_walks, mutation):
    changed = 0
    for name, args, res in host_walks:
        changed += changed_clear_slots(res, IW.walk(*args, mutations=(mutation,)))
    print(f"mutation {mutation}: {changed} clear slots change on the constructed states")
    assert changed >= MUTATION_MINIMUM


# On the recorded frames the branches behind these mutations occur; the others need states real streams rarely make.
@pytest.mark.parametrize("mutation", ["second_into_original", "no_depth_reread", "stale_candidates", "raw_positions",
                                      "drop_secondary", "no_detach"])
def test_mutations_show_on_the_recorded_frames(golden, mutation):
    changed = 0
    for f in (5, 6, 7):
        _, _, res = golden_walk(golden, f)
        _, _, mutated = golden_walk(golden, f, (mutation,))
        changed += changed_clear_slots(res, mutated)
    print(f"mutation {mutation}: {changed} clear slots change on golden frames 5-7")
    assert changed >= 1
