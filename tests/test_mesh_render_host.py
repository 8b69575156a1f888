"""sm_render_mesh on the CPU: the plain-C restatement (tests/mesh_render_walk.c) against float64 geometry. Watertight
coverage of grids and fans, perspective-correct depth and colour, independence of winding and corner rotation, the
disk fallback of an empty list, and the golden f7 state under its own mesh. The GPU kernels are compared with the
restatement bit for bit in tests/test_mesh_render_gpu.py."""
import numpy as np
import pytest

from surfelmeshing_b200 import _lib
from tests import mesh_render_walk as MRW
from tests import mesh_walk as M
from tests import render_walk
from tests.test_render_host import make_rows

# fx = fy = 64 and c = 0.5 put the screen point of (k / 64, l / 64, 1) exactly on the centre of pixel (k, l)
W, H = 96, 80
CAM = dict(width=W, height=H, fx=64.0, fy=64.0, cx=0.5, cy=0.5)
IDENTITY = np.eye(4, dtype=np.float32)[:3]
EPS = 2.0 ** -24


def vertex_rows(points, colors=None):
    """A [25, n] state whose slots are the given points (facing the camera, radius 0.01, colour per point)."""
    points = np.asarray(points, np.float64)
    if colors is None:
        colors = [(int(37 * i) % 256, int(91 * i) % 256, int(13 * i) % 256) for i in range(len(points))]
    return make_rows([(tuple(p), (0, 0, -1), 0.01, tuple(c)) for p, c in zip(points, colors)])


def walk(rows, tris, T=IDENTITY, near=0.1, far=10.0, disks=False, cam=CAM, stats=False):
    return MRW.render(rows, tris, T, cam["width"], cam["height"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], near,
                      far, unmeshed_surfels=disks, stats=stats)


def pixel_centres():
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64) + 0.5, np.arange(W, dtype=np.float64) + 0.5, indexing="ij")
    return xs, ys


def grid_mesh(nx, ny, step, origin, diagonal, z=1.0):
    """Vertices on a regular screen grid (in pixels, through pixel centres when `step` and `origin` are integers) at
    depth z, each quad split along `diagonal` ("/", "\\" or "alternate"). Returns (points, triangles, boundary)."""
    pts = [((origin[0] + i * step) / 64.0 * z, (origin[1] + j * step) / 64.0 * z, z) for j in range(ny) for i in range(nx)]
    tris = []
    for j in range(ny - 1):
        for i in range(nx - 1):
            a, b, c, d = j * nx + i, j * nx + i + 1, (j + 1) * nx + i + 1, (j + 1) * nx + i
            slash = diagonal == "/" or (diagonal == "alternate" and (i + j) % 2 == 0)
            tris += [(a, b, c), (a, c, d)] if slash else [(a, b, d), (b, c, d)]
    lo = (origin[0] + 0.5, origin[1] + 0.5)
    hi = (origin[0] + 0.5 + (nx - 1) * step, origin[1] + 0.5 + (ny - 1) * step)
    return pts, np.array(tris), (lo, hi)


@pytest.mark.parametrize("diagonal", ["/", "\\", "alternate"])
@pytest.mark.parametrize("step,origin", [(5, (3, 4)), (3.7, (2.3, 1.9))], ids=["on_pixel_centres", "off_centre"])
def test_grid_is_watertight(diagonal, step, origin):
    pts, tris, (lo, hi) = grid_mesh(17, 14, step, origin, diagonal)
    rng = np.random.default_rng(7)
    perm = rng.permutation(len(pts))            # slot order unrelated to the grid
    rows = vertex_rows(np.asarray(pts)[np.argsort(perm)])
    out = walk(rows, perm[tris])
    xs, ys = pixel_centres()
    inside = (xs > lo[0]) & (xs < hi[0]) & (ys > lo[1]) & (ys < hi[1])
    covered = out["index"] != MRW.INVALID
    assert inside.sum() > 1000
    assert covered[inside].all(), f"{int((inside & ~covered).sum())} holes"
    # nothing outside the closed rectangle
    outside = (xs < lo[0]) | (xs > hi[0]) | (ys < lo[1]) | (ys > hi[1])
    assert not covered[outside].any()
    assert np.allclose(out["depth"][covered], 1.0, rtol=4 * EPS, atol=0)


def point_in_polygon(xs, ys, poly):
    """float64 even-odd test and the distance of each point to the polygon's boundary."""
    inside = np.zeros(xs.shape, bool)
    dist = np.full(xs.shape, np.inf)
    for (x0, y0), (x1, y1) in zip(poly, np.roll(poly, -1, axis=0)):
        cond = (y0 > ys) != (y1 > ys)
        with np.errstate(divide="ignore", invalid="ignore"):
            xcross = (x1 - x0) * (ys - y0) / (y1 - y0) + x0
        inside ^= cond & (xs < xcross)
        ex, ey = x1 - x0, y1 - y0
        t = np.clip(((xs - x0) * ex + (ys - y0) * ey) / (ex * ex + ey * ey), 0, 1)
        dist = np.minimum(dist, np.hypot(xs - (x0 + t * ex), ys - (y0 + t * ey)))
    return inside, dist


def fan(rng, k, centre, jitter):
    angles = np.sort(rng.uniform(0, 2 * np.pi, k)) if jitter else np.linspace(0, 2 * np.pi, k, endpoint=False)
    radii = rng.uniform(12, 35, k) if jitter else np.full(k, 30.0)
    ring = np.stack([centre[0] + radii * np.cos(angles), centre[1] + radii * np.sin(angles)], 1)
    return ring


@pytest.mark.parametrize("seed", range(12))
def test_fans_are_watertight(seed):
    rng = np.random.default_rng(seed)
    k = int(rng.integers(3, 14)) if seed else 8
    centre = np.array([48.0, 40.0]) if seed % 3 == 0 else rng.uniform([40, 34], [56, 46])
    ring = fan(rng, k, centre, jitter=seed > 0)
    if seed > 0:   # the screen points go through fp32 arithmetic on the way, so ask for a convex-enough star
        angles = np.sort(np.arctan2(ring[:, 1] - centre[1], ring[:, 0] - centre[0]))
        if np.max(np.diff(np.append(angles, angles[0] + 2 * np.pi))) >= 0.9 * np.pi:
            pytest.skip("not a star polygon about its centre")
    z = rng.uniform(0.8, 2.5, k + 1) if seed % 2 else np.ones(k + 1)
    screen = np.vstack([centre, ring])
    pts = [((u - 0.5) / 64.0 * zz, (v - 0.5) / 64.0 * zz, zz) for (u, v), zz in zip(screen, z)]
    perm = rng.permutation(k + 1)
    rows = vertex_rows(np.asarray(pts)[np.argsort(perm)])
    tris = np.array([(0, 1 + i, 1 + (i + 1) % k) for i in range(k)])
    if seed % 4 == 1:
        tris = tris[:, ::-1]                     # clockwise on screen
    tris = perm[tris]
    out = walk(rows, tris)
    xs, ys = pixel_centres()
    inside, dist = point_in_polygon(xs, ys, ring)
    clear = inside & (dist > 1e-3)
    covered = out["index"] != MRW.INVALID
    assert clear.sum() > 200
    assert covered[clear].all(), f"{int((clear & ~covered).sum())} holes in a fan of {k}"
    assert not covered[~inside & (dist > 1e-3)].any()


def plane_depth(dx, dy, p0, normal):
    """float64 depth along the ray (dx, dy, 1) to the plane through p0 with the given normal."""
    return (normal @ p0) / (normal[0] * dx + normal[1] * dy + normal[2])


def slanted_quad(colors):
    p = np.array([[-0.3, -0.25, 1.2], [0.35, -0.2, 2.6], [0.3, 0.3, 2.4], [-0.35, 0.25, 1.1]], np.float32)
    # put the fourth corner on the plane of the first three (in float64 of the float32 coordinates)
    n = np.cross(p[1].astype(np.float64) - p[0], p[2].astype(np.float64) - p[0])
    p[3, 2] = np.float32(p[0, 2] - (n[0] * (p[3, 0] - p[0, 0]) + n[1] * (p[3, 1] - p[0, 1])) / n[2])
    cam = dict(width=W, height=H, fx=70.0, fy=72.0, cx=48.3, cy=39.6)
    return p, vertex_rows(p, colors), np.array([(0, 1, 2), (0, 2, 3)]), cam


def test_slanted_plane_depth_matches_float64():
    p, rows, tris, cam = slanted_quad(None)
    out = walk(rows, tris, cam=cam)
    covered = out["index"] != MRW.INVALID
    assert covered.sum() > 500
    ys, xs = np.nonzero(covered)
    dx = (xs + 0.5 - cam["cx"]) / cam["fx"]
    dy = (ys + 0.5 - cam["cy"]) / cam["fy"]
    p64 = p.astype(np.float64)
    normal = np.cross(p64[1] - p64[0], p64[2] - p64[0])
    want = plane_depth(dx, dy, p64[0], normal)
    got = out["depth"][covered].astype(np.float64)
    # Bound: the screen points carry ~3 eps * |u| each; an edge value ~4 eps * S with S = the sum of the magnitudes of
    # its two products (<= 2 * L * R, L the longest edge, R the largest |coordinate| including the pixel); a weight
    # b = w / D then errs by delta_b = (3 eps R L + 8 eps L R) / |D| + 2 eps, and 1 / sum(b_k / z_k) by at most
    # 3 delta_b z_max / z_min relative, plus 4 eps for the last divisions.
    u = cam["fx"] * p64[:, 0] / p64[:, 2] + cam["cx"]
    v = cam["fy"] * p64[:, 1] / p64[:, 2] + cam["cy"]
    R = max(np.abs(u).max(), np.abs(v).max(), W, H)
    L = max(np.hypot(u[i] - u[j], v[i] - v[j]) for i in range(4) for j in range(i))
    D = min(abs((u[b] - u[a]) * (v[c] - v[a]) - (v[b] - v[a]) * (u[c] - u[a])) for a, b, c in tris)
    delta_b = 11 * EPS * R * L / D + 2 * EPS
    bound = (3 * delta_b * p64[:, 2].max() / p64[:, 2].min() + 4 * EPS) * want
    err = np.abs(got - want)
    print(f"slanted plane: max |dz| / bound = {float((err / bound).max()):.3f}, max rel {float((err / want).max()):.2e}")
    assert np.all(err <= bound)


def test_vertex_pixels_have_the_vertex_colour():
    pts, tris, _ = grid_mesh(9, 8, 6, (10, 9), "alternate", z=1.0)
    pts = [(x * (1 + 0.1 * (i % 3)), y * (1 + 0.1 * (i % 3)), 1 + 0.1 * (i % 3)) for i, (x, y, _) in enumerate(pts)]
    rng = np.random.default_rng(3)
    colors = [tuple(int(c) for c in rng.integers(0, 256, 3)) for _ in pts]
    rows = vertex_rows(pts, colors)
    out = walk(rows, tris)
    for i, (x, y, z) in enumerate(pts):
        u = 64.0 * np.float32(np.float32(x) / np.float32(z)) + 0.5
        v = 64.0 * np.float32(np.float32(y) / np.float32(z)) + 0.5
        px, py = int(np.floor(u)), int(np.floor(v))
        if abs(u - px - 0.5) > 1e-6 or abs(v - py - 0.5) > 1e-6:
            continue   # the fp32 screen point is not exactly a pixel centre
        assert out["index"][py, px] != MRW.INVALID
        assert tuple(out["color"][py, px]) == colors[i], (i, out["color"][py, px], colors[i])


def test_two_colour_quad_matches_float64_interpolation():
    a, b = (230, 10, 40), (5, 120, 250)
    p, rows, tris, cam = slanted_quad([a, a, b, b])
    out = walk(rows, tris, cam=cam)
    covered = out["index"] != MRW.INVALID
    ys, xs = np.nonzero(covered)
    p64 = p.astype(np.float64)
    u = cam["fx"] * p64[:, 0] / p64[:, 2] + cam["cx"]
    v = cam["fy"] * p64[:, 1] / p64[:, 2] + cam["cy"]
    X, Y = xs + 0.5, ys + 0.5
    cols = np.array([a, a, b, b], np.float64)
    want = np.zeros((len(X), 3))
    done = np.zeros(len(X), bool)
    for t, (i, j, k) in enumerate(tris):
        D = (u[j] - u[i]) * (v[k] - v[i]) - (v[j] - v[i]) * (u[k] - u[i])
        wi = ((u[k] - u[j]) * (Y - v[j]) - (v[k] - v[j]) * (X - u[j])) / D
        wj = ((u[i] - u[k]) * (Y - v[k]) - (v[i] - v[k]) * (X - u[k])) / D
        wk = 1 - wi - wj
        sel = (out["index"][ys, xs] == t)
        q = np.stack([wi / p64[i, 2], wj / p64[j, 2], wk / p64[k, 2]], 1)
        want[sel] = (q @ cols[[i, j, k]])[sel] / q.sum(1)[sel, None]
        done |= sel
    assert done.all() and len(X) > 500
    diff = np.abs(out["color"][ys, xs].astype(np.float64) - want)
    print(f"two-colour quad: max |colour - float64| = {diff.max():.3f}")
    assert diff.max() <= 1.0


def test_winding_and_rotation_do_not_matter():
    p = [(-0.2, -0.15, 1.3), (0.25, -0.1, 2.1), (0.05, 0.3, 1.7)]
    rows = vertex_rows(p, [(250, 0, 0), (0, 250, 0), (0, 0, 250)])
    cam = dict(width=W, height=H, fx=70.0, fy=-72.0, cx=48.3, cy=39.6)
    outs = [walk(rows, [order], cam=cam) for order in
            [(0, 1, 2), (1, 2, 0), (2, 0, 1), (0, 2, 1), (2, 1, 0), (1, 0, 2)]]
    assert (outs[0]["index"] == 0).sum() > 100
    for o in outs[1:]:
        for k in ("depth", "color", "normal", "index"):
            assert np.array_equal(o[k].view(np.uint8), outs[0][k].view(np.uint8)), k
    n = outs[0]["normal"][outs[0]["index"] == 0]
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-6) and np.all(n[:, 2] < 0)   # faces the camera


def test_empty_list_with_the_flag_is_the_disk_render():
    rows = make_rows([((0.0, 0.0, 2.0), (0, 0, -1), 0.3, (50, 0, 0)), ((0.1, 0.05, 1.8), (0.2, 0, -1), 0.2, (0, 50, 0)),
                      ((0.0, 0.0, 2.0), (0, 0, -1), -0.5, (9, 9, 9))])
    cam = dict(width=64, height=48, fx=50.0, fy=50.0, cx=32.25, cy=24.25)
    ref = render_walk.render(rows, IDENTITY, 64, 48, 50.0, 50.0, 32.25, 24.25, 0.1, 10.0)
    out = walk(rows, np.zeros((0, 3), np.int64), disks=True, cam=cam)
    for k in ("depth", "color", "normal"):
        assert np.array_equal(out[k].view(np.uint8), ref[k].view(np.uint8)), k
    valid = ref["index"] != MRW.INVALID
    assert valid.sum() > 100
    assert np.array_equal(out["index"][valid], ref["index"][valid] | MRW.DISK)
    assert np.all(out["index"][~valid] == MRW.INVALID)
    empty = walk(rows, np.zeros((0, 3), np.int64), disks=False, cam=cam)
    assert np.all(empty["index"] == MRW.INVALID) and np.all(empty["depth"] == 0)


def test_triangles_win_ties_against_disks_and_stale_corners_are_skipped():
    pts = [(-0.2, -0.2, 1.0), (0.3, -0.2, 1.0), (0.0, 0.3, 1.0), (0.05, 0.0, 1.0)]
    rows = vertex_rows(pts)
    rows[7, 3] = 0.3 ** 2                          # slot 3: a disk in the triangle's plane, not a corner
    out = walk(rows, [(0, 1, 2), (0, 1, 9), (0, 1, 2)], disks=True, cam=dict(CAM, cx=48.0, cy=40.0))
    tri = out["index"] == 0
    disk = out["index"] == (MRW.DISK | 3)
    assert tri.sum() > 100 and disk.sum() > 100    # the disk shows only outside the triangle
    assert not np.any(out["index"] == 1) and not np.any(out["index"] == 2)   # stale corner; the duplicate loses
    rows[7, 2] = -rows[7, 2]                       # merge a corner: the triangle goes, its live corners become disks
    out = walk(rows, [(0, 1, 2)], disks=True, cam=dict(CAM, cx=48.0, cy=40.0))
    assert not np.any(out["index"] == 0)
    assert set(np.unique(out["index"]).tolist()) <= {MRW.DISK | 0, MRW.DISK | 1, MRW.DISK | 3, MRW.INVALID}


def test_golden_state_under_its_own_mesh():
    from tests.util import GOLDEN_DIR
    meta = np.load(GOLDEN_DIR / "golden_320x240_meta.npz")
    w, h, fx, fy, cx, cy = [float(v) for v in meta["camera"]]
    rows = M.golden_f7()
    tris, stats, _ = M.triangulate(rows)
    T = meta["frame_T_global"][7]
    cam = dict(width=int(w), height=int(h), fx=fx, fy=fy, cx=cx, cy=cy)
    out, st = walk(rows, tris.astype(np.int64), T=T, near=0.1, far=100.0, disks=True, cam=cam, stats=True)
    idx = out["index"]
    tri = (idx != MRW.INVALID) & (idx < MRW.DISK)
    disk = (idx != MRW.INVALID) & (idx >= MRW.DISK)
    print(f"golden f7: {len(tris)} triangles, {st['triangles']} drawn, {st['disks']} disks; coverage "
          f"{tri.mean():.3f} by triangles + {disk.mean():.3f} by disks")
    assert tri.mean() > 0.1 and st["marked"] == stats["vertices_meshed"]
    assert np.all(out["depth"][tri | disk] > 0)


def test_header_declares_the_call():
    assert "sm_render_mesh" in _lib.EXPORTED_SYMBOLS and _lib.RENDER_UNMESHED_SURFELS == 1
