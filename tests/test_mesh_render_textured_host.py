"""The plain-C restatement of sm_render_mesh_textured (tests/mesh_render_textured_walk.c, rule T8) against a float64
numpy statement of T8 on the texture tests' hand-built scenes and on random atlases, and its exact properties: a
constant atlas, lookups at texel centres, unusable and out-of-range uv, winding and rotation, and every output but
the triangles' colour equal to sm_render_mesh's."""
import numpy as np
import pytest

from surfelmeshing_b200._lib import TextureParams
from tests import mesh_render_textured_walk as MRTW
from tests import mesh_render_walk as MRW
from tests import texture_walk as TW

NEAR, FAR = 0.1, 10.0
CAM = TW.CAM


def walk(rows, tris, texture, T, cam=CAM, disks=True):
    return MRTW.render_textured(rows, tris, texture, T, near=NEAR, far=FAR, unmeshed_surfels=disks, **cam)


def plain(rows, tris, T, cam=CAM, disks=True):
    return MRW.render(rows, tris, T, near=NEAR, far=FAR, unmeshed_surfels=disks, **cam)


def triangle_pixels(out):
    return (out["index"] != MRW.INVALID) & (out["index"] < MRW.DISK)


def t8_float64(rows, tris, texture, T, cam, index):
    """T8 in float64 at every pixel whose winning key is a triangle (given by `index`): the perspective-correct
    barycentrics of the pixel centre, the uv of each corner, the clamp and the bilinear lookup. Returns the colour
    [N, 3] (float64, before rounding) and the pixel coordinates."""
    atlas, uv = texture
    atlas = atlas.astype(np.float64)
    uv = np.asarray(uv, np.float64).reshape(-1, 3, 2)
    H, W = atlas.shape[:2]
    ys, xs = np.nonzero((index != MRW.INVALID) & (index < MRW.DISK))
    t = index[ys, xs].astype(np.int64)
    tri = np.asarray(tris, np.int64).reshape(-1, 3)[t]
    Tm = np.asarray(T, np.float64).reshape(3, 4)
    P = rows[3:6].astype(np.float64).T
    c = np.einsum("ij,nkj->nki", Tm[:, :3], P[tri]) + Tm[:, 3]
    u = cam["fx"] * c[..., 0] / c[..., 2] + cam["cx"]
    v = cam["fy"] * c[..., 1] / c[..., 2] + cam["cy"]
    x, y = xs + 0.5, ys + 0.5

    def edge(j, k):
        return (u[:, k] - u[:, j]) * (y - v[:, j]) - (v[:, k] - v[:, j]) * (x - u[:, j])
    w = np.stack([edge(1, 2), edge(2, 0), edge(0, 1)], 1)   # affine weights, any winding
    q = w / c[..., 2]
    b = q / q.sum(1, keepdims=True)                          # perspective-correct barycentrics
    U = np.einsum("nk,nkc->nc", b, uv[t])
    U = np.clip(U, 0.0, 1.0)
    fx_, fy_ = U[:, 0] * W - 0.5, U[:, 1] * H - 0.5
    x0, y0 = np.floor(fx_).astype(int), np.floor(fy_).astype(int)
    ax, ay = (fx_ - x0)[:, None], (fy_ - y0)[:, None]

    def at(i, j):
        return atlas[np.clip(j, 0, H - 1), np.clip(i, 0, W - 1)]
    top = at(x0, y0) + ax * (at(x0 + 1, y0) - at(x0, y0))
    bot = at(x0, y0 + 1) + ax * (at(x0 + 1, y0 + 1) - at(x0, y0 + 1))
    return top + ay * (bot - top), ys, xs


def assert_close_to_float64(rows, tris, texture, T, cam=CAM, disks=True):
    out = walk(rows, tris, texture, T, cam, disks)
    sample, ys, xs = t8_float64(rows, tris, texture, T, cam, out["index"])
    want = np.minimum(np.floor(sample + 0.5), 255)
    diff = np.abs(out["color"][ys, xs].astype(np.float64) - want)
    assert len(ys) > 100
    assert diff.max() <= 1, (diff.max(), (diff > 0).mean())
    return out


def assert_same_but_colour(out, ref):
    for k in ("depth", "normal", "index"):
        assert np.array_equal(out[k].view(np.uint32), ref[k].view(np.uint32)), k
    other = ~triangle_pixels(ref)
    assert np.array_equal(out["color"][other], ref["color"][other])


def scenes():
    """name -> (rows, triangles, views for texture_walk.texture, render pose)."""
    cam, I = CAM, TW.identity()
    quad = TW.quad_rows()
    front = TW.quad_rows(z=1.0, half=0.2, grid=2, color=(0, 0, 255))
    back = TW.quad_rows(z=2.0, half=0.6, grid=4, color=(0, 255, 0))
    tilted = TW.look_from((0.4, 0.2, 0.1), (0.0, 0.0, 1.0))
    return {
        "quad_ramp": (*quad, [TW.View(cam, I, TW.ramp(cam))], I),
        "quad_ramp_tilted": (*quad, [TW.View(cam, I, TW.ramp(cam))], tilted),
        "stack_two_views": (*TW.stack(front, back), [TW.View(cam, I, TW.ramp(cam)),
                                                    TW.View(cam, tilted, TW.ramp(cam)[::-1])],
                            TW.look_from((-0.3, 0.1, 0.0))),
        "quad_solid": (*quad, [TW.View(cam, I, TW.solid(cam, (12, 200, 99)))], tilted),
    }


SCENES = scenes()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_walk_matches_float64_on_textured_scenes(name):
    rows, tris, views, T = SCENES[name]
    atlas, uv, _ = TW.texture(rows, tris, views, TextureParams.defaults(texel_size=0.005))
    out = assert_close_to_float64(rows, tris, (atlas, uv), T)
    assert_same_but_colour(out, plain(rows, tris, T))


def random_texture(rng, count, W, H, lo=0.0, hi=1.0):
    atlas = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    uv = rng.uniform(lo, hi, (count, 3, 2)).astype(np.float32)
    return atlas, uv


@pytest.mark.parametrize("seed,size", [(0, (37, 23)), (1, (1, 1)), (2, (1, 64)), (3, (256, 8))])
def test_walk_matches_float64_on_random_atlases(seed, size):
    rng = np.random.default_rng(seed)
    rows, tris = TW.stack(TW.quad_rows(grid=6), TW.quad_rows(z=1.5, half=0.5, grid=3, offset=(0.2, 0.1)))
    W, H = size
    texture = random_texture(rng, len(tris), W, H, -0.1, 1.1)
    for T in (TW.identity(), TW.look_from((0.3, -0.2, 0.0))):
        out = assert_close_to_float64(rows, tris, texture, T)
        assert_same_but_colour(out, plain(rows, tris, T))


def test_constant_atlas_gives_its_colour():
    rng = np.random.default_rng(7)
    rows, tris = TW.quad_rows(grid=5)
    atlas = np.broadcast_to(np.array([17, 230, 101], np.uint8), (9, 13, 3)).copy()
    uv = rng.uniform(-2.0, 3.0, (len(tris), 3, 2)).astype(np.float32)
    out = walk(rows, tris, (atlas, uv), TW.look_from((0.2, 0.3, 0.1)))
    tri = triangle_pixels(out)
    assert tri.sum() > 500
    assert (out["color"][tri] == [17, 230, 101]).all()


def test_texel_centres_return_their_texel():
    rng = np.random.default_rng(8)
    rows, tris = TW.quad_rows(grid=4)
    W, H = 16, 8
    atlas = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    i, j = rng.integers(0, W, len(tris)), rng.integers(0, H, len(tris))
    centre = np.stack([(i + 0.5) / W, (j + 0.5) / H], 1).astype(np.float32)
    uv = np.repeat(centre[:, None, :], 3, axis=1)
    out = walk(rows, tris, (atlas, uv), TW.identity())
    tri = triangle_pixels(out)
    t = out["index"][tri].astype(np.int64)
    assert np.array_equal(out["color"][tri], atlas[j[t], i[t]])


def test_nan_uv_takes_the_vertex_colour():
    rng = np.random.default_rng(9)
    rows, tris = TW.quad_rows(grid=4)
    rows[24] = rng.integers(0, 1 << 24, rows.shape[1]).astype(np.uint32).view(np.float32)
    atlas, uv = random_texture(rng, len(tris), 8, 8)
    bad = np.arange(len(tris)) % 3 == 0
    uv[bad, 1, 0] = np.nan
    uv[np.arange(len(tris)) % 3 == 1, 2, 1] = np.inf
    bad |= np.arange(len(tris)) % 3 == 1
    T = TW.look_from((0.1, 0.1, 0.0))
    out, ref = walk(rows, tris, (atlas, uv), T), plain(rows, tris, T)
    tri = triangle_pixels(ref)
    on_bad = tri & bad[np.where(tri, ref["index"], 0).astype(np.int64)]
    assert on_bad.sum() > 100 and (tri & ~on_bad).sum() > 100
    assert np.array_equal(out["color"][on_bad], ref["color"][on_bad])
    assert not np.array_equal(out["color"][tri & ~on_bad], ref["color"][tri & ~on_bad])


def test_uv_outside_the_unit_square_clamps():
    rng = np.random.default_rng(10)
    rows, tris = TW.quad_rows(grid=3)
    W, H = 11, 7
    atlas = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    uv = np.empty((len(tris), 3, 2), np.float32)
    uv[..., 0], uv[..., 1] = 1.5, -3.0          # U clamps to 1 (the last column), V to 0 (the first row)
    out = walk(rows, tris, (atlas, uv), TW.identity())
    tri = triangle_pixels(out)
    assert (out["color"][tri] == atlas[0, W - 1]).all()
    uv[..., 0], uv[..., 1] = -1e30, 7.0         # the first column, the last row
    out = walk(rows, tris, (atlas, uv), TW.identity())
    assert (out["color"][tri] == atlas[H - 1, 0]).all()


def test_rotating_or_rewinding_with_the_uv_changes_nothing():
    rng = np.random.default_rng(11)
    rows, tris = TW.stack(TW.quad_rows(grid=5), TW.quad_rows(z=1.4, half=0.5, grid=3))
    texture = random_texture(rng, len(tris), 29, 17)
    T = TW.look_from((0.2, -0.1, 0.05))
    ref = walk(rows, tris, texture, T)
    atlas, uv = texture
    for order in ((1, 2, 0), (2, 0, 1), (0, 2, 1), (2, 1, 0)):
        out = walk(rows, tris[:, order], (atlas, uv[:, order]), T)
        for k in ref:
            assert np.array_equal(out[k].view(np.uint8), ref[k].view(np.uint8)), (order, k)


@pytest.mark.parametrize("disks", [True, False])
def test_only_the_triangle_colour_differs_from_render(disks):
    rng = np.random.default_rng(12)
    rows, tris = TW.stack(TW.quad_rows(grid=4), TW.quad_rows(z=2.0, half=0.8, grid=2))
    # slots no triangle names, drawn as disks with the flag, and stale triangles
    extra = TW.quad_rows(z=1.2, half=0.1, grid=1, offset=(0.4, 0.3))[0]
    rows = np.concatenate([rows, extra], axis=1)
    n = rows.shape[1]
    tris = np.concatenate([tris, [[0, 1, n + 3], [2, 3, n]]])
    texture = random_texture(rng, len(tris), 20, 20)
    T = TW.look_from((-0.2, 0.1, 0.0))
    out, ref = walk(rows, tris, texture, T, disks=disks), plain(rows, tris, T, disks=disks)
    assert_same_but_colour(out, ref)
    assert ((ref["index"] >= MRW.DISK) & (ref["index"] != MRW.INVALID)).any() == disks


def test_empty_list_with_an_empty_atlas():
    rows, _ = TW.quad_rows(grid=2)
    empty = np.zeros((0, 3), np.int64)
    texture = (np.zeros((0, 0, 3), np.uint8), np.zeros((0, 3, 2), np.float32))
    out, ref = walk(rows, empty, texture, TW.identity()), plain(rows, empty, TW.identity())
    for k in ref:
        assert np.array_equal(out[k].view(np.uint8), ref[k].view(np.uint8)), k
