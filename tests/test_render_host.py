"""sm_render_surfels on the CPU: the plain-C restatement (tests/render_walk.c) against float64 geometry, its tie and
merge rules, and the layout of sm_render_params. The GPU kernels are compared with the restatement bit for bit in
tests/test_render_gpu.py."""
import ctypes as C

import numpy as np

from surfelmeshing_b200 import _lib
from tests import render_walk

W, H = 64, 48
FX = FY = 50.0
CX, CY = 32.25, 24.25           # no pixel centre lies on the optical axis
IDENTITY = np.eye(4, dtype=np.float32)[:3]


def make_rows(disks):
    """[25, n] float32 state of disks given as (centre, normal, radius, rgb); radius < 0 marks a merged slot."""
    rows = np.zeros((_lib.ROW_COUNT, len(disks)), np.float32)
    rows.view(np.uint32)[19:23] = 0xFFFFFFFF
    for i, (c, n, r, rgb) in enumerate(disks):
        n = np.asarray(n, np.float64)
        n = n / np.linalg.norm(n)
        rows[0:3, i] = c
        rows[3:6, i] = c
        rows[6, i] = 1.0
        rows[7, i] = np.float32(r) * np.float32(r) * (1 if r > 0 else -1)
        rows[8:11, i] = n
        rows.view(np.uint32)[24, i] = rgb[0] | (rgb[1] << 8) | (rgb[2] << 16)
    return rows


def walk(rows, T=IDENTITY, near=0.1, far=10.0, w=W, h=H):
    return render_walk.render(rows, T, w, h, FX, FY, CX, CY, near, far)


def ray_grid(w=W, h=H):
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    return (xs + 0.5 - CX) / FX, (ys + 0.5 - CY) / FY


def analytic_cover(c, n, r):
    """float64: covered mask and the squared distance of each pixel ray's plane hit from the centre."""
    dx, dy = ray_grid()
    c, n = np.asarray(c, np.float64), np.asarray(n, np.float64) / np.linalg.norm(n)
    den = n[0] * dx + n[1] * dy + n[2]
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (n @ c) / den
    d2 = (t * dx - c[0]) ** 2 + (t * dy - c[1]) ** 2 + (t - c[2]) ** 2
    d2 = np.where(np.isfinite(t) & (t > 0), d2, np.inf)
    return d2 <= r * r, d2


def test_head_on_disk_covers_the_projected_circle():
    c, r = (0.05, -0.03, 2.0), 0.4
    out = walk(make_rows([(c, (0, 0, -1), r, (10, 20, 30))]))
    dx, dy = ray_grid()
    # the disk faces the camera: a pixel is covered iff its centre's ray meets the plane z = 2 inside the circle
    dist = np.hypot(2.0 * dx - c[0], 2.0 * dy - c[1])
    clear = np.abs(dist - r) > 1e-4
    inside = dist <= r
    assert inside.sum() > 300
    assert np.array_equal((out["index"] == 0)[clear], inside[clear])
    assert np.all(out["index"][~inside & clear] == 0xFFFFFFFF)
    assert np.allclose(out["depth"][inside], 2.0, rtol=0, atol=1e-6)
    assert np.all(out["depth"][~inside & clear] == 0)
    assert np.all(out["color"][inside] == (10, 20, 30)) and np.all(out["color"][~inside & clear] == 0)
    assert np.allclose(out["normal"][inside], (0, 0, -1))


def test_tilted_disk_covers_an_ellipse():
    c, n, r = (-0.1, 0.05, 1.5), (0.6, -0.2, -0.75), 0.35
    out = walk(make_rows([(c, n, r, (1, 2, 3))]))
    cover, d2 = analytic_cover(c, n, r)
    clear = np.abs(d2 - r * r) > 1e-5
    assert cover.sum() > 200
    assert np.array_equal((out["index"] == 0)[clear], cover[clear])
    # the depth is the plane hit along the pixel's ray
    dx, dy = ray_grid()
    nn = np.asarray(n) / np.linalg.norm(n)
    t = (nn @ np.asarray(c)) / (nn[0] * dx + nn[1] * dy + nn[2])
    assert np.allclose(out["depth"][cover & clear], t[cover & clear], rtol=1e-5)


def test_edge_on_disk_covers_nothing():
    out = walk(make_rows([((0.0, 0.0, 2.0), (1, 0, 0), 0.5, (9, 9, 9))]))
    assert np.all(out["index"] == 0xFFFFFFFF) and np.all(out["depth"] == 0)


def test_ties_go_to_the_lower_slot_and_the_nearer_disk_wins():
    disk = ((0.0, 0.0, 2.0), (0, 0, -1), 0.3, (50, 0, 0))
    out = walk(make_rows([disk, ((0.0, 0.0, 2.0), (0, 0, -1), 0.3, (0, 50, 0))]))
    covered = out["index"] != 0xFFFFFFFF
    assert covered.sum() > 100 and np.all(out["index"][covered] == 0)
    out = walk(make_rows([disk, ((0.0, 0.0, 1.9), (0, 0, -1), 0.1, (0, 0, 50))]))
    near = out["index"] == 1
    assert near.sum() > 10 and np.all(out["color"][near] == (0, 0, 50)) and np.allclose(out["depth"][near], 1.9)


def test_merged_slots_and_depth_range_are_skipped():
    rows = make_rows([((0.0, 0.0, 2.0), (0, 0, -1), -0.5, (1, 1, 1)),    # merged: radius^2 < 0
                      ((0.0, 0.0, 2.0), (0, 0, -1), 0.2, (2, 2, 2)),
                      ((0.0, 0.0, -2.0), (0, 0, 1), 0.5, (3, 3, 3)),     # behind the camera
                      ((0.0, 0.0, 20.0), (0, 0, -1), 5.0, (4, 4, 4))])   # beyond far
    out = walk(rows)
    assert set(np.unique(out["index"]).tolist()) == {1, 0xFFFFFFFF}
    out = walk(rows, near=2.5)
    assert np.all(out["index"] == 0xFFFFFFFF)


def test_disk_around_the_camera_plane_is_clipped_by_the_ray_test():
    """A disk whose bounding sphere reaches z = 0 tests the whole image; only hits with t > 0 count."""
    out = walk(make_rows([((0.0, 0.0, 0.2), (0, 0.3, -1), 1.0, (7, 7, 7))]))
    cover, _ = analytic_cover((0.0, 0.0, 0.2), (0, 0.3, -1), 1.0)
    assert cover.all() and np.all(out["index"] == 0)


def test_render_params_layout():
    p = _lib.RenderParams
    assert C.sizeof(p) == 32
    assert [(name, getattr(p, name).offset) for name, _ in p._fields_] == [
        ("width", 0), ("height", 4), ("fx", 8), ("fy", 12), ("cx", 16), ("cy", 20), ("near_depth", 24),
        ("far_depth", 28)]
