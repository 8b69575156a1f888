"""sm_mesh_texture on the GPU: atlas, uv and stats bit-equal to the plain-C restatement (tests/texture_walk.c) on the
host cases, golden f7 (with its fill, and simplified) and a 48-frame VGA stream with every 4th frame as a view;
read-only behaviour, commutation with sm_compact, the capacity protocol, argument and input errors, the OBJ export,
and the colour error on held-out frames against per-vertex colour."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, mesh_io, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import SimplifyParams, TextureParams, TextureStats, TextureViewDesc
from tests import texture_walk as TW
from tests import test_mesh_texture_host as HOST
from tests.test_mesh_gpu import loaded, run_stream

pytestmark = pytest.mark.gpu


def gpu_view(v):
    cam = S.Camera(v.cam["width"], v.cam["height"], v.cam["fx"], v.cam["fy"], v.cam["cx"], v.cam["cy"])
    return R.TextureView(torch.as_tensor(v.color, device="cuda"), cam, view_T_global=v.T, near=v.near, far=v.far)


def assert_same(rec, rows, tris, views, params):
    want_atlas, want_uv, want_stats = TW.texture(rows, tris, views, params)
    t = torch.as_tensor(np.asarray(tris, np.int64).reshape(-1, 3).astype(np.int32), device="cuda")
    atlas, uv, stats = rec.texture_mesh(t, [gpu_view(v) for v in views], params)
    torch.cuda.synchronize()
    assert TW.stats_dict(stats) == want_stats
    assert np.array_equal(atlas.cpu().numpy(), want_atlas)
    assert np.array_equal(uv.cpu().numpy().view(np.uint32), want_uv.view(np.uint32))
    return want_stats


def host_cases():
    cam, I = TW.CAM, TW.identity()
    quad = TW.quad_rows()
    front = TW.quad_rows(z=1.0, half=0.2, grid=2, color=(0, 0, 255))
    back = TW.quad_rows(z=2.0, half=0.6, grid=4, color=(0, 0, 255))
    narrow, wide = dict(cam, fx=400.0, fy=400.0), dict(cam, fx=40.0, fy=40.0)
    grazing = TW.look_from((2.0, 0.0, 0.65), (0.0, 0.0, 1.0))
    p01 = TextureParams.defaults(texel_size=0.01)
    soup = HOST.random_soup()
    return {
        "soup": (soup, [], p01),
        "constant": (quad, [TW.View(cam, I, TW.solid(cam, (12, 200, 99)))], p01),
        "ramp": (quad, [TW.View(cam, I, TW.ramp(cam))], p01),
        "occlusion": (TW.stack(front, back), [TW.View(narrow, I, TW.solid(narrow, (255, 0, 0))),
                                             TW.View(wide, I, TW.solid(wide, (0, 255, 0)))], p01),
        "grazing": (quad, [TW.View(cam, grazing, TW.solid(cam, (255, 255, 255)))], p01),
        "grazing_89": (quad, [TW.View(cam, grazing, TW.solid(cam, (255, 255, 255)))],
                       TextureParams.defaults(texel_size=0.01, max_view_angle_deg=89.0)),
        "fallback": (TW.quad_rows(grid=3), [TW.View(cam, TW.look_from((0.0, 0.0, 3.0), (0.0, 0.0, 5.0)),
                                                    TW.solid(cam, (255, 255, 255)))],
                     TextureParams.defaults(texel_size=0.02)),
        "ramp_and_tilted": (quad, [TW.View(cam, I, TW.ramp(cam)),
                                   TW.View(cam, TW.look_from((0.4, 0.2, 0.1), (0.0, 0.0, 1.0)), TW.ramp(cam)[::-1])],
                            TextureParams.defaults(texel_size=0.005, depth_tolerance=0.02)),
    }


CASES = host_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_bit_equal_on_the_host_cases(name):
    (rows, tris), views, params = CASES[name]
    rec = loaded(rows)
    s = assert_same(rec, rows, tris, views, params)
    assert s["texels"] > 0
    rec.close()


@pytest.mark.parametrize("mesh", ["full_with_fill", "simplified"])
def test_bit_equal_on_golden_f7(mesh):
    rows, meshes = HOST.golden_meshes()
    rec = loaded(rows)
    s = assert_same(rec, rows, meshes[mesh], HOST.golden_views(), HOST.GOLDEN_PARAMS)
    assert s["texels_seen"] > 0.5 * s["texels"]
    rec.close()


def stream_views(st, frames, near=0.1, far=20.0):
    cam = st.camera
    return [R.TextureView(st.color[f], cam, view_T_global=st.frame_T_global[f], near=near, far=far) for f in frames]


def host_views(st, frames, near=0.1, far=20.0):
    cam = dict(width=st.camera.width, height=st.camera.height, fx=st.camera.fx, fy=st.camera.fy, cx=st.camera.cx,
               cy=st.camera.cy)
    return [TW.View(cam, st.frame_T_global[f], st.color[f].cpu().numpy(), near, far) for f in frames]


@pytest.fixture(scope="module")
def vga():
    """The cloud after the 48-frame VGA stream, its mesh with the fill, and that mesh simplified."""
    cam = S.Camera.tum(640, 480)
    rec, st = run_stream(cam, 48)
    full = rec.triangulate()[0]
    full = torch.cat([full, rec.fill_holes(full)[0]])
    simple, _ = rec.simplify_mesh(full, SimplifyParams.defaults())
    torch.cuda.synchronize()
    yield rec, st, full, simple
    rec.close()


def test_bit_equal_on_the_vga_stream(vga):
    rec, st, full, simple = vga
    rows, _, _ = rec.dump_state()
    first, last = st.integrated_range()
    frames = list(range(first, last, 4))
    p = TextureParams.defaults()
    for tri in (simple, full):
        want_atlas, want_uv, want_stats = TW.texture(rows, tri.cpu().numpy(), host_views(st, frames), p)
        atlas, uv, stats = rec.texture_mesh(tri, stream_views(st, frames), p)
        torch.cuda.synchronize()
        print(f"VGA stream, {len(tri)} triangles, {len(frames)} views: {TW.stats_dict(stats)}")
        assert TW.stats_dict(stats) == want_stats
        assert np.array_equal(atlas.cpu().numpy(), want_atlas)
        assert np.array_equal(uv.cpu().numpy().view(np.uint32), want_uv.view(np.uint32))


def test_read_only(vga):
    rec, st, full, simple = vga
    before, n, merges = rec.dump_state()
    first, last = st.integrated_range()
    rec.texture_mesh(simple, stream_views(st, range(first, last, 8)))
    after, n2, merges2 = rec.dump_state()
    assert (n2, merges2) == (n, merges)
    assert np.array_equal(before.view(np.uint32), after.view(np.uint32))


def test_commutes_with_compaction():
    rec, st = run_stream(S.Camera.tum(320, 240), 48)
    _, _, merges = rec.dump_state()
    assert merges > 0
    tri = rec.triangulate()[0]
    tri = torch.cat([tri, rec.fill_holes(tri)[0]])
    first, last = st.integrated_range()
    views = stream_views(st, range(first, last, 6))
    p = TextureParams.defaults(texel_size=0.008)
    atlas, uv, stats = rec.texture_mesh(tri, views, p)
    _, m = rec.compact(return_map=True)
    mapped = R.remap_triangles(tri, m)
    assert len(mapped) == len(tri)
    atlas2, uv2, stats2 = rec.texture_mesh(mapped, views, p)
    assert TW.stats_dict(stats2) == TW.stats_dict(stats)
    assert torch.equal(atlas2, atlas) and torch.equal(uv2.view(torch.int32), uv.view(torch.int32))
    rec.close()


def test_errors_write_nothing_and_capacity_protocol():
    (rows, tris), views, p = CASES["constant"]
    rec = loaded(rows)
    want_atlas, want_uv, want_stats = TW.texture(rows, tris, views, p)
    H, W = want_atlas.shape[:2]
    fn = rec.lib.fn["mesh_texture"]
    gv = [gpu_view(v) for v in views]
    descs = (TextureViewDesc * 1)(gv[0].desc())
    src = torch.as_tensor(tris.astype(np.int32), device="cuda")
    atlas = torch.full((H + 2, W + 4, 3), 7, dtype=torch.uint8, device="cuda")
    uv = torch.full((len(tris) + 1, 3, 2), -7.0, device="cuda")
    stats = TextureStats()

    def call(t=src, params=p, d=descs, count=None, nv=1, a=atlas, pitch=None, cw=None, ch=None, u=uv, st=stats):
        if not isinstance(t, torch.Tensor):
            t = torch.as_tensor(np.asarray(t, np.int32).reshape(-1, 3), device="cuda")
        status = fn(rec._h, None, C.byref(params) if params is not None else None,
                    C.c_void_p(t.data_ptr()) if t is not None else None, len(t) if count is None else count, d, nv,
                    C.c_void_p(a.data_ptr()) if a is not None else None,
                    a.stride(0) if (a is not None and pitch is None) else (pitch or 0),
                    (a.shape[1] if a is not None else 0) if cw is None else cw,
                    (a.shape[0] if a is not None else 0) if ch is None else ch,
                    C.c_void_p(u.data_ptr()) if u is not None else None, C.byref(st) if st is not None else None)
        torch.cuda.synchronize()
        return status

    def with_camera(**kw):
        d = TextureViewDesc.from_buffer_copy(descs[0])
        for k, v in kw.items():
            if k in ("color", "color_pitch"):
                setattr(d, k, v)
            elif k == "pose":
                d.view_T_global[0] = v
            else:
                setattr(d.camera, k, v)
        return (TextureViewDesc * 1)(d)

    launches = rec.lib.fn["kernel_launch_count"]()
    for bad in (TextureParams.defaults(texel_size=0.0), TextureParams.defaults(texel_size=float("nan")),
                TextureParams.defaults(texel_size=float("inf")), TextureParams.defaults(max_atlas_side=4),
                TextureParams.defaults(max_atlas_side=65536), TextureParams.defaults(max_view_angle_deg=0.0),
                TextureParams.defaults(max_view_angle_deg=90.5), TextureParams.defaults(depth_tolerance=-0.1),
                TextureParams.defaults(depth_tolerance=float("nan"))):
        assert call(params=bad) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(params=None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(st=None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert fn(rec._h, None, C.byref(p), None, 3, descs, 1, None, 0, 0, 0, None, C.byref(stats)) == \
        _lib.SM_ERR_INVALID_ARGUMENT
    assert call(count=1 << 28) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(d=None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(nv=_lib.TEXTURE_MAX_VIEWS + 1) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(nv=-1) == _lib.SM_ERR_INVALID_ARGUMENT
    for kw in (dict(width=0), dict(fx=0.0), dict(cx=float("inf")), dict(near_depth=0.0), dict(far_depth=0.05),
               dict(pose=float("nan")), dict(color=None), dict(color_pitch=3 * TW.CAM["width"] - 1)):
        assert call(d=with_camera(**kw)) == _lib.SM_ERR_INVALID_ARGUMENT, kw
    assert call(a=None, cw=W, ch=H) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(cw=-1) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(pitch=3 * (W + 4) - 1) == _lib.SM_ERR_INVALID_ARGUMENT
    assert call(u=src) == _lib.SM_ERR_INVALID_ARGUMENT                              # uv overlaps triangles
    assert call(u=atlas[1:]) == _lib.SM_ERR_INVALID_ARGUMENT                        # uv overlaps the atlas
    assert rec.lib.fn["kernel_launch_count"]() == launches
    n = rows.shape[1]
    for t in ([[0, 1, n]], [[0, 0, 1]]):
        assert call(np.concatenate([tris, t])) == _lib.SM_ERR_INVALID_ARGUMENT
        assert TW.stats_dict(stats) == dict.fromkeys(TW.STATS, 0)
    assert call(np.concatenate([tris, [[0, 1, n]]])) == _lib.SM_ERR_INVALID_ARGUMENT
    assert rec.lib.fn["last_error"]() == b"sm_mesh_texture: a corner is not a present slot below surfels_size()"
    assert (atlas == 7).all() and (uv == -7.0).all()
    # a layout query, a capacity one texel short each way, max_atlas_side, then enough
    layout = dict(want_stats, texels_seen=0, texels_fallback=0, views_used=0)
    assert call(a=None) == _lib.SM_ERR_CAPACITY and TW.stats_dict(stats) == layout
    assert call(cw=W - 1) == _lib.SM_ERR_CAPACITY and TW.stats_dict(stats) == layout
    assert rec.lib.fn["last_error"]() == \
        f"sm_mesh_texture: a {W} x {H} atlas does not fit the capacity of {W - 1} x {H + 2}".encode()
    assert call(ch=H - 1) == _lib.SM_ERR_CAPACITY and TW.stats_dict(stats) == layout
    assert call(params=TextureParams.defaults(texel_size=p.texel_size, max_atlas_side=W - 1)) == _lib.SM_ERR_CAPACITY
    assert rec.lib.fn["last_error"]() == \
        f"sm_mesh_texture: the atlas needs a side of {W} texels, above max_atlas_side {W - 1}; raise texel_size".encode()
    assert (atlas == 7).all() and (uv == -7.0).all()
    assert call() == _lib.SM_OK and TW.stats_dict(stats) == want_stats
    got = atlas.cpu().numpy()
    assert np.array_equal(got[:H, :W], want_atlas) and (got[H:] == 7).all() and (got[:, W:] == 7).all()
    assert np.array_equal(uv[:len(tris)].cpu().numpy(), want_uv) and (uv[len(tris):] == -7.0).all()
    assert call(u=None) == _lib.SM_OK                                                # uv may be NULL
    assert call(np.zeros((0, 3)), a=None) == _lib.SM_OK and stats.atlas_width == 0
    rec.close()


def test_obj_export(tmp_path):
    rec, st = run_stream(S.Camera.tum(320, 240), 16, stream_id=3)
    first, last = st.integrated_range()
    views = stream_views(st, range(first, last, 3))
    p = TextureParams.defaults(texel_size=0.01)
    rec.save_mesh_obj(tmp_path / "plain.obj")
    rec.save_mesh_obj(tmp_path / "tex.obj", texture=p, views=views)
    tri, _ = rec.triangulate()
    atlas, uv, _ = rec.texture_mesh(tri, views, p)
    v, _, faces = mesh_io.read_obj(tmp_path / "tex.obj")
    v0, _, faces0 = mesh_io.read_obj(tmp_path / "plain.obj")
    assert np.array_equal(v, v0) and np.array_equal(faces, faces0)
    vt, fvt, mtllib = mesh_io.read_obj_texcoords(tmp_path / "tex.obj")
    assert mtllib == "tex.mtl" and "map_Kd tex.png" in (tmp_path / "tex.mtl").read_text()
    assert np.allclose(vt[fvt.ravel(), 0], uv[..., 0].cpu().numpy().ravel(), atol=1e-7)
    assert np.array_equal(mesh_io.read_png(tmp_path / "tex.png"), atlas.cpu().numpy())
    rec.close()


def sample_atlas(atlas, uv):
    """Bilinear lookups (texel centres at integer + 0.5, clamped to the atlas) at uv points [N, 2] -> [N, 3]."""
    H, W = atlas.shape[:2]
    x, y = uv[:, 0] * W - 0.5, uv[:, 1] * H - 0.5
    x0, y0 = np.floor(x).astype(int), np.floor(y).astype(int)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    a = atlas.astype(np.float64)

    def at(i, j):
        return a[np.clip(j, 0, H - 1), np.clip(i, 0, W - 1)]
    top = at(x0, y0) * (1 - fx) + at(x0 + 1, y0) * fx
    bot = at(x0, y0 + 1) * (1 - fx) + at(x0 + 1, y0 + 1) * fx
    return top * (1 - fy) + bot * fy


def colour_errors(rec, st, tri, atlas, uv, frames):
    """Median absolute colour error (per channel, over the pixels where render_mesh hits a triangle) on the frames,
    of the atlas sampled at the pixel's surface point and of render_mesh's per-vertex colour; then the two means."""
    rows, _, _ = rec.dump_state()
    cam = st.camera
    P = rows[3:6].T.astype(np.float64)
    tri_np = tri.cpu().numpy()
    atlas, uv = atlas.cpu().numpy(), uv.cpu().numpy().astype(np.float64)
    tex_err, vert_err = [], []
    for f in frames:
        out = rec.render_mesh(tri, st.frame_T_global[f], cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy,
                              near=0.1, far=20.0, unmeshed_surfels=False, outputs=("color", "index"))
        index = out["index"].cpu().numpy()
        color = out["color"].cpu().numpy().astype(np.float64)
        truth = st.color[f].cpu().numpy().astype(np.float64)
        ys, xs = np.nonzero(index >= 0)
        t = index[ys, xs]
        # barycentrics of the pixel ray's hit on the triangle, in the camera frame
        Tm = np.asarray(st.frame_T_global[f], np.float64)
        corners = np.einsum("ij,tkj->tki", Tm[:, :3], P[tri_np[t]]) + Tm[:, 3]
        ray = np.stack([(xs + 0.5 - cam.cx) / cam.fx, (ys + 0.5 - cam.cy) / cam.fy, np.ones(len(xs))], 1)
        e1, e2 = corners[:, 1] - corners[:, 0], corners[:, 2] - corners[:, 0]
        n = np.cross(e1, e2)
        depth = np.einsum("ij,ij->i", n, corners[:, 0]) / np.einsum("ij,ij->i", n, ray)
        hit = ray * depth[:, None] - corners[:, 0]
        # solve hit = b1 e1 + b2 e2 in the least-squares sense
        G = np.stack([e1, e2], 2)
        b = np.linalg.solve(np.einsum("nki,nkj->nij", G, G), np.einsum("nki,nk->ni", G, hit)[..., None])[..., 0]
        b = np.clip(b, 0, 1)
        w = np.stack([1 - b[:, 0] - b[:, 1], b[:, 0], b[:, 1]], 1)
        point_uv = np.einsum("nk,nkc->nc", w, uv[t])
        tex = sample_atlas(atlas, point_uv)
        tex_err.append(np.abs(tex - truth[ys, xs]).ravel())
        vert_err.append(np.abs(color[ys, xs] - truth[ys, xs]).ravel())
    tex_err, vert_err = np.concatenate(tex_err), np.concatenate(vert_err)
    return (float(np.median(tex_err)), float(np.median(vert_err)), float(tex_err.mean()), float(vert_err.mean()))


def test_texture_beats_vertex_colour_on_held_out_frames(vga):
    rec, st, full, simple = vga
    first, last = st.integrated_range()
    views = list(range(first, last, 4))
    held_out = [f for f in range(first + 2, last, 8)]
    p = TextureParams.defaults()
    # Margins fixed from the first run on an H100 (DESIGN.md section 5.15): on the simplified mesh the median is 0
    # against 1; on the full mesh both medians are 0 (a triangle covers about one pixel), so the means decide there.
    for name, tri in (("simplified", simple), ("full", full)):
        atlas, uv, stats = rec.texture_mesh(tri, stream_views(st, views), p)
        tex, vert, tex_mean, vert_mean = colour_errors(rec, st, tri, atlas, uv, held_out)
        print(f"{name}: {len(tri)} triangles, atlas {stats.atlas_width} x {stats.atlas_height}, "
              f"seen {stats.texels_seen} / {stats.texels}; held-out median |error|: textured {tex:.2f}, "
              f"per-vertex {vert:.2f}; mean: textured {tex_mean:.3f}, per-vertex {vert_mean:.3f}")
        if name == "simplified":
            assert tex < vert - 0.5
        else:
            assert tex <= vert and tex_mean < vert_mean
