"""sm_mesh_texture's rules (X1-X8 of include/surfel_b200.h) through the plain-C restatement (tests/texture_walk.c),
checked against properties stated independently here: the layout (squares disjoint, aligned, inside the atlas, in
class order) and the footprint of every UV triangle, the class boundaries, colours from constant and ramp views,
occlusion, the angle cut, the corner-blend fallback, golden f7 with its fill and simplified, and the OBJ + MTL + PNG
writers."""

import numpy as np
import pytest

from surfelmeshing_b200 import mesh_io
from surfelmeshing_b200._lib import SimplifyParams, TextureParams
from tests import mesh_walk as M
from tests import simplify_walk as SW
from tests import texture_walk as TW


def squares_from_uv(uv, W, H):
    """Per triangle (s, x0, y0, half) read back from its uv (X4): half 0 has two corners on its square's left
    column x0 + 1, half 1 two on its right column x0 + s - 1."""
    X = np.rint(uv[..., 0].astype(np.float64) * W).astype(np.int64)
    Y = np.rint(uv[..., 1].astype(np.float64) * H).astype(np.int64)
    out = []
    for x, y in zip(X, Y):
        lo, hi = x.min(), x.max()
        s = int(hi - lo + 4)
        half = 0 if (x == lo).sum() == 2 else 1
        x0 = int(lo - 1) if half == 0 else int(hi - s + 1)
        y0 = int(y.min() - 1) if half == 0 else int(y.max() - s + 1)
        out.append((s, x0, y0, half))
    return np.array(out, np.int64).reshape(-1, 4)


def morton(x, y):
    code = 0
    for b in range(20):
        code |= ((x >> b) & 1) << (2 * b) | ((y >> b) & 1) << (2 * b + 1)
    return code


def check_layout(uv, stats, rng, samples=24):
    W, H = stats["atlas_width"], stats["atlas_height"]
    T = len(uv)
    sq = squares_from_uv(uv, W, H)
    s, x0, y0, half = sq.T
    assert set(np.unique(s)) <= {8, 16, 32, 64, 128, 256, 512}
    assert np.all(x0 % s == 0) and np.all(y0 % s == 0)                                  # aligned
    assert np.all(x0 >= 0) and np.all(y0 >= 0) and np.all(x0 + s <= W) and np.all(y0 + s <= H)
    assert W & (W - 1) == 0 and W * W >= sum((s[half == 0] ** 2)) and (W // 2) ** 2 < sum(s[half == 0] ** 2)
    assert H == (y0 + s).max()
    # class order: by (s descending, t ascending), consecutive pairs share a square, squares at rising Morton codes
    order = np.lexsort((np.arange(T), -s))
    keys = [(int(s[t]), int(x0[t]), int(y0[t])) for t in order]
    sorted_s = s[order]
    for k, t in enumerate(order):
        r = k - int(np.searchsorted(-sorted_s, -s[t]))   # rank within the class
        partner = k + 1 if r % 2 == 0 else k - 1
        assert half[t] == r % 2
        if partner < T and sorted_s[partner] == s[t]:
            assert keys[partner] == keys[k]
    firsts = [t for t in order if half[t] == 0]
    codes = [morton(int(x0[t]), int(y0[t])) for t in firsts]
    area = np.cumsum([0] + [int(s[t]) ** 2 for t in firsts])[:-1]
    assert codes == list(area)                                                          # running area offsets
    # disjoint: every texel of the atlas belongs to at most one square
    owner = np.full((H, W), -1, np.int64)
    for k, t in enumerate(firsts):
        block = owner[y0[t]:y0[t] + s[t], x0[t]:x0[t] + s[t]]
        assert (block == -1).all()
        block[:] = k
    # the bilinear footprint of points inside each UV triangle stays in its half
    for t in range(T):
        w = rng.dirichlet((1, 1, 1), samples)
        w = np.vstack([w, np.eye(3), [[0.5, 0.5, 0], [0, 0.5, 0.5], [0.5, 0, 0.5]]])
        pts = w @ (uv[t].astype(np.float64) * [W, H])
        i0 = np.floor(pts - 0.5).astype(np.int64)
        for dx in (0, 1):
            for dy in (0, 1):
                li, lj = i0[:, 0] + dx - x0[t], i0[:, 1] + dy - y0[t]
                assert np.all((li >= 0) & (lj >= 0) & (li < s[t]) & (lj < s[t]))
                assert np.all(li + lj <= s[t] - 1) if half[t] == 0 else np.all(li + lj >= s[t])
    return sq


def random_soup(count=300, seed=3):
    """Triangles of many sizes (2 cm .. 6 m legs) over a random cloud: every tile class and a few clamped ones."""
    rng = np.random.default_rng(seed)
    pts, tris = [], []
    for t in range(count):
        size = 10 ** rng.uniform(-1.7, 0.8)
        o = rng.uniform(-1, 1, 3) + [0, 0, 3]
        a, b = rng.normal(size=3), rng.normal(size=3)
        pts += [o, o + size * a / np.linalg.norm(a), o + size * b / np.linalg.norm(b)]
        tris.append((3 * t, 3 * t + 1 + t % 2, 3 * t + 2 - t % 2))
    return M.make_rows(pts, (0.0, 0.0, -1.0), 1e-4), np.array(tris)


def test_layout_of_a_soup_of_sizes():
    rows, tris = random_soup()
    p = TextureParams.defaults(texel_size=0.01)
    atlas, uv, stats = TW.texture(rows, tris, [], p)
    assert stats["triangles"] == len(tris) and stats["tiles_clamped"] > 0
    sq = check_layout(uv, stats, np.random.default_rng(0))
    assert len(np.unique(sq[:, 0])) == 7
    # no views: every texel takes the corner blend; texels outside every half-tile stay 0
    assert stats["texels_fallback"] == stats["texels"] and stats["texels_seen"] == 0 and stats["views_used"] == 0
    s, half = sq[:, 0], sq[:, 3]
    assert stats["texels"] == sum(int(x) * (int(x) + 1) // 2 if h == 0 else int(x) * (int(x) - 1) // 2
                                  for x, h in zip(s, half))
    painted = np.zeros(atlas.shape[:2], bool)
    for (sz, x0, y0, h) in sq:
        i, j = np.meshgrid(np.arange(sz), np.arange(sz), indexing="xy")
        own = (i + j <= sz - 1) if h == 0 else (i + j >= sz)
        painted[y0:y0 + sz, x0:x0 + sz] |= own
    assert not atlas[~painted].any()


@pytest.mark.parametrize("texel", [0.25, 0.01])
def test_class_boundaries_and_clamp(texel):
    """Right isosceles triangles with legs exactly (s - 4) * texel_size (binary exact with texel 0.25) take class s;
    one ulp longer takes 2 s; past (512 - 4) * texel_size the tile is capped and counted."""
    legs, want = [], []
    for s in (8, 16, 32, 64, 128, 256, 512):
        L = np.float32((s - 4) * texel)
        legs += [L, np.nextafter(L, np.float32(np.inf))]
        want += [s, min(2 * s, 512)]
    pts, tris = [], []
    for k, L in enumerate(legs):
        o = np.array([0.0, 0.0, 1.0 + k], np.float32)
        pts += [o, o + np.array([L, 0, 0], np.float32), o + np.array([0, L, 0], np.float32)]
        tris.append((3 * k + 1, 3 * k + 2, 3 * k))   # a (opposite the hypotenuse) listed last
    rows = M.make_rows(pts, (0.0, 0.0, -1.0), 1e-4)
    p = TextureParams.defaults(texel_size=texel, max_atlas_side=32768)
    _, uv, stats = TW.texture(rows, np.array(tris), [], p)
    sq = check_layout(uv, stats, np.random.default_rng(1), samples=4)
    exact = texel == 0.25
    if exact:
        assert list(sq[:, 0]) == want
    assert stats["tiles_clamped"] == (1 if exact else sum(1 for L in legs if np.float32(L) > np.float32(508 * texel)))
    # the corner opposite the longest edge sits at (1, 1) of half 0 / (s - 1, s - 1) of half 1
    W, H = stats["atlas_width"], stats["atlas_height"]
    for t, (s, x0, y0, half) in enumerate(sq):
        a = np.rint(uv[t, 2] * [W, H]).astype(int)
        assert tuple(a) == ((x0 + 1, y0 + 1) if half == 0 else (x0 + s - 1, y0 + s - 1))


def texel_points(rows, tris, uv, stats):
    """Per texel of every half-tile, restated in float64 from the uv: (atlas y, x, triangle, alpha, beta, X)."""
    W, H = stats["atlas_width"], stats["atlas_height"]
    sq = squares_from_uv(uv, W, H)
    out = []
    for t, (s, x0, y0, half) in enumerate(sq):
        tri = np.asarray(tris[t])
        # which listed corner is a: the one at the square's (1, 1) or (s - 1, s - 1)
        X = np.rint(uv[t] * [W, H]).astype(int)
        ka = int(np.flatnonzero((X[:, 0] == (x0 + 1 if half == 0 else x0 + s - 1)) &
                                (X[:, 1] == (y0 + 1 if half == 0 else y0 + s - 1)))[0])
        a, b, c = (rows[3:6, tri[(ka + k) % 3]].astype(np.float64) for k in range(3))
        for j in range(s):
            for i in range(s):
                if (i + j > s - 1) if half == 0 else (i + j < s):
                    continue
                x, y = i + 0.5, j + 0.5
                al, be = ((x - 1) / (s - 4), (y - 1) / (s - 4)) if half == 0 else \
                    ((s - 1 - x) / (s - 4), (s - 1 - y) / (s - 4))
                al, be = max(al, 0.0), max(be, 0.0)
                if al + be > 1:
                    al = al / (al + be)
                    be = 1 - al
                out.append((y0 + j, x0 + i, t, al, be, a + al * (b - a) + be * (c - a)))
    return out


def test_constant_view_gives_its_colour_exactly():
    rows, tris = TW.quad_rows()
    view = TW.View(TW.CAM, TW.identity(), TW.solid(TW.CAM, (12, 200, 99)))
    atlas, uv, stats = TW.texture(rows, tris, [view], TextureParams.defaults(texel_size=0.01))
    assert stats["texels_seen"] > 0.5 * stats["texels"] and stats["views_used"] == 1
    seen_color = np.all(atlas == (12, 200, 99), axis=2)
    assert seen_color.sum() == stats["texels_seen"]


def test_ramp_view_is_followed_within_one_step():
    rows, tris = TW.quad_rows()
    cam = TW.CAM
    view = TW.View(cam, TW.identity(), TW.ramp(cam))
    atlas, uv, stats = TW.texture(rows, tris, [view], TextureParams.defaults(texel_size=0.01))
    checked = 0
    for y, x, t, al, be, X in texel_points(rows, tris, uv, stats):
        u = cam["fx"] * X[0] / X[2] + cam["cx"] - 0.5
        v = cam["fy"] * X[1] / X[2] + cam["cy"] - 0.5
        inside = 25 <= u + 0.5 <= 71 and 17 <= v + 0.5 <= 63   # a pixel inside the quad's image, [24, 72] x [16, 64]
        if atlas[y, x, 2] != 77:                               # the corner blend (blue 50): not seen
            assert not inside
            continue
        want = (2 * u, 3 * v, 77)
        assert np.all(np.abs(atlas[y, x].astype(float) - want) <= 1.0), (atlas[y, x], want)
        checked += 1
    assert checked == stats["texels_seen"] and checked > 1000


def test_occlusion():
    """View 1 (red, narrow) sees only the front quad; view 2 (green, wide) sees both: the back quad is pure green
    wherever it is seen."""
    front = TW.quad_rows(z=1.0, half=0.2, grid=2, color=(0, 0, 255))
    back = TW.quad_rows(z=2.0, half=0.6, grid=4, color=(0, 0, 255))
    rows, tris = TW.stack(front, back)
    n_front = len(front[1])
    narrow = dict(TW.CAM, fx=400.0, fy=400.0)
    wide = dict(TW.CAM, fx=40.0, fy=40.0)
    views = [TW.View(narrow, TW.identity(), TW.solid(narrow, (255, 0, 0))),
             TW.View(wide, TW.identity(), TW.solid(wide, (0, 255, 0)))]
    atlas, uv, stats = TW.texture(rows, tris, views, TextureParams.defaults(texel_size=0.01))
    assert stats["views_used"] == 2
    back_seen = front_mixed = 0
    for y, x, t, al, be, X in texel_points(rows, tris, uv, stats):
        c = tuple(atlas[y, x])
        if t >= n_front and c != (0, 0, 255) and c[2] == 0:
            assert c == (0, 255, 0)
            back_seen += 1
        if t < n_front and c[0] > 0 and c[1] > 0:
            front_mixed += 1
    assert back_seen > 1000 and front_mixed > 100


def test_grazing_view_contributes_nothing():
    rows, tris = TW.quad_rows()
    T = TW.look_from((2.0, 0.0, 0.65), (0.0, 0.0, 1.0))   # about 80 degrees from the quad's normal
    view = TW.View(TW.CAM, T, TW.solid(TW.CAM, (255, 255, 255)))
    _, _, stats = TW.texture(rows, tris, [view], TextureParams.defaults(texel_size=0.01))
    assert stats["texels_seen"] == 0 and stats["views_used"] == 0
    _, _, wide = TW.texture(rows, tris, [view], TextureParams.defaults(texel_size=0.01, max_view_angle_deg=89.0))
    assert wide["texels_seen"] > 0 and wide["views_used"] == 1


def test_fallback_is_the_corner_blend():
    """Texels no view sees take ((1 - a - b) C_a + a C_b) + b C_c of the corner colours (rounded half up)."""
    rows, tris = TW.quad_rows(grid=3)
    rows.view(np.uint32)[24] = (np.arange(rows.shape[1], dtype=np.uint32) * 2654435761) & 0xFFFFFF
    behind = TW.look_from((0.0, 0.0, 3.0), (0.0, 0.0, 5.0))   # sees nothing of the quad
    view = TW.View(TW.CAM, behind, TW.solid(TW.CAM, (255, 255, 255)))
    atlas, uv, stats = TW.texture(rows, tris, [view], TextureParams.defaults(texel_size=0.02))
    assert stats["texels_fallback"] == stats["texels"] and stats["views_used"] == 0
    rgb = rows.view(np.uint32)[24]
    for y, x, t, al, be, X in texel_points(rows, tris, uv, stats):
        W, H = stats["atlas_width"], stats["atlas_height"]
        Xc = np.rint(uv[t] * [W, H]).astype(int)
        sq = squares_from_uv(uv[t:t + 1], W, H)[0]
        ka = int(np.flatnonzero((Xc[:, 0] == (sq[1] + 1 if sq[3] == 0 else sq[1] + sq[0] - 1)) &
                                (Xc[:, 1] == (sq[2] + 1 if sq[3] == 0 else sq[2] + sq[0] - 1)))[0])
        corners = [int(tris[t][(ka + k) % 3]) for k in range(3)]
        for ch in range(3):
            c = [float((rgb[s] >> (8 * ch)) & 0xFF) for s in corners]
            want = (1 - al - be) * c[0] + al * c[1] + be * c[2]
            assert abs(int(atlas[y, x, ch]) - want) <= 0.5 + 1e-3


def golden_views(count=4):
    from tests.util import GOLDEN_DIR, load_npz_xz
    meta = np.load(GOLDEN_DIR / "golden_320x240_meta.npz")
    w, h, fx, fy, cx, cy = [float(v) for v in meta["camera"]]
    cam = dict(width=int(w), height=int(h), fx=fx, fy=fy, cx=cx, cy=cy)
    color = load_npz_xz(GOLDEN_DIR / "golden_320x240_inputs_a.npz.xz")["color"]
    frames = np.linspace(1, len(color) - 2, count).astype(int)
    return [TW.View(cam, meta["frame_T_global"][f], color[f], near=0.1, far=20.0) for f in frames]


GOLDEN_PARAMS = TextureParams.defaults(texel_size=0.02)


def golden_meshes():
    rows = M.golden_f7()
    full = SW.meshed(rows)
    simple, _ = SW.simplify(rows, full, SimplifyParams.defaults())
    return rows, {"full_with_fill": full, "simplified": simple}


@pytest.mark.parametrize("mesh", ["full_with_fill", "simplified"])
def test_golden_f7(mesh):
    rows, meshes = golden_meshes()
    tris = meshes[mesh]
    atlas, uv, stats = TW.texture(rows, tris, golden_views(), GOLDEN_PARAMS)
    print(f"golden f7 {mesh}: {stats}")
    assert stats["texels_seen"] + stats["texels_fallback"] == stats["texels"]
    assert stats["texels_seen"] > 0.5 * stats["texels"] and stats["views_used"] == 4
    check_layout(uv, stats, np.random.default_rng(2), samples=2)


def test_input_errors_and_empty_list():
    rows, tris = TW.quad_rows(grid=1)
    for bad in ([[0, 1, rows.shape[1]]], [[0, 0, 1]]):
        with pytest.raises(ValueError):
            TW.texture(rows, np.concatenate([tris, bad]), [])
    merged = rows.copy()
    merged[7, 3] = -1.0
    with pytest.raises(ValueError):
        TW.texture(merged, tris, [])
    atlas, uv, stats = TW.texture(rows, np.zeros((0, 3)), [])
    assert atlas.shape == (0, 0, 3) and uv.shape == (0, 3, 2) and stats["atlas_width"] == 0


def test_too_wide_for_max_atlas_side():
    rows, tris = random_soup(40)
    p = TextureParams.defaults(texel_size=0.001, max_atlas_side=256)
    atlas, uv, stats = TW.texture(rows, tris, [], p)
    assert atlas is None and stats["atlas_width"] > 256


def test_obj_mtl_png_round_trip(tmp_path):
    rows, tris = TW.quad_rows(grid=2)
    rows.view(np.uint32)[24] = (np.arange(rows.shape[1], dtype=np.uint32) * 2654435761) & 0xFFFFFF
    atlas, uv, stats = TW.texture(rows, tris, [], TextureParams.defaults(texel_size=0.02))
    positions = rows[3:6].T.copy()
    colors = rows.view(np.uint32)[24].view(np.uint8).reshape(-1, 4)[:, :3]
    plain, again = tmp_path / "plain.obj", tmp_path / "again.obj"
    mesh_io.write_obj(plain, positions, colors, tris)
    mesh_io.write_obj(again, positions, colors, tris, uvs=None, material=None)
    assert plain.read_bytes() == again.read_bytes() and b"vt" not in plain.read_bytes()
    obj = tmp_path / "mesh.obj"
    mesh_io.write_png(tmp_path / "mesh.png", atlas)
    mesh_io.write_mtl(tmp_path / "mesh.mtl", "mesh.png")
    assert mesh_io.write_obj(obj, positions, colors, tris, uvs=uv, material="mesh.mtl") == (len(positions), len(tris))
    v, c, faces = mesh_io.read_obj(obj)
    assert np.allclose(v, positions, atol=1e-5) and np.array_equal(faces, tris)
    vt, fvt, mtllib = mesh_io.read_obj_texcoords(obj)
    assert mtllib == "mesh.mtl" and np.array_equal(fvt, np.arange(3 * len(tris)).reshape(-1, 3))
    assert np.allclose(vt[:, 0], uv[..., 0].ravel(), atol=1e-7) and np.allclose(1 - vt[:, 1], uv[..., 1].ravel(), atol=1e-7)
    assert np.array_equal(mesh_io.read_png(tmp_path / "mesh.png"), atlas)
    mtl = (tmp_path / "mesh.mtl").read_text()
    assert "newmtl atlas" in mtl and "map_Kd mesh.png" in mtl
    rng = np.random.default_rng(4)
    odd = rng.integers(0, 256, (7, 5, 3), dtype=np.uint8)
    mesh_io.write_png(tmp_path / "odd.png", odd)
    assert np.array_equal(mesh_io.read_png(tmp_path / "odd.png"), odd)


def test_png_reader_takes_every_row_filter(tmp_path):
    """A PNG whose rows use filters 1-4 (as other writers produce) reads back to the same image."""
    import struct
    import zlib
    rng = np.random.default_rng(9)
    img = rng.integers(0, 256, (5, 4, 3)).astype(np.int64)
    rows = []
    prev = np.zeros(12, np.int64)
    for y in range(5):
        cur = img[y].reshape(-1)
        kind = y % 5
        a = np.concatenate([[0, 0, 0], cur[:-3]])
        c = np.concatenate([[0, 0, 0], prev[:-3]])
        if kind == 0:
            pred = np.zeros(12, np.int64)
        elif kind == 1:
            pred = a
        elif kind == 2:
            pred = prev
        elif kind == 3:
            pred = (a + prev) // 2
        else:
            p = a + prev - c
            pa, pb, pc = np.abs(p - a), np.abs(p - prev), np.abs(p - c)
            pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, prev, c))
        rows.append(bytes([kind]) + ((cur - pred) & 0xFF).astype(np.uint8).tobytes())
        prev = cur
    chunk = mesh_io._png_chunk
    data = (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", 4, 5, 8, 2, 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(b"".join(rows))) + chunk(b"IEND", b""))
    (tmp_path / "f.png").write_bytes(data)
    assert np.array_equal(mesh_io.read_png(tmp_path / "f.png"), img.astype(np.uint8))
