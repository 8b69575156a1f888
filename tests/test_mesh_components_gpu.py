"""sm_mesh_components on the GPU: out, labels, table and stats bit-equal to the plain-C restatement
(tests/components_walk.c) on the host cases, golden f7 (with its fill, and simplified) and a 48-frame VGA stream;
read-only behaviour, labels and table after sm_compact + remap_triangles, the output taken by sm_mesh_simplify,
sm_mesh_texture and sm_render_mesh, the capacity protocol, argument and input errors, and the OBJ export."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, mesh_io, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import ComponentParams, ComponentStats, HoleParams, SimplifyParams, TextureParams
from tests import components_walk as CW
from tests import mesh_walk as M
from tests import simplify_walk as SW
from tests import test_mesh_components_host as HOST
from tests.test_mesh_gpu import loaded, run_stream

pytestmark = pytest.mark.gpu


def dev(tri):
    return torch.as_tensor(np.asarray(tri, np.int64).reshape(-1, 3).astype(np.int32), device="cuda")


def raw_table(table):
    """The table dict of mesh_components() as TABLE_DTYPE records."""
    P = len(table["triangles"])
    out = np.zeros(P, CW.TABLE_DTYPE)
    for k in ("triangles", "area", "lo", "hi", "first_triangle"):
        out[k] = table[k].cpu().numpy()
    out["kept"] = table["kept"].cpu().numpy().astype(np.int32)
    return out


def assert_same(rec, rows, tri, p):
    want_out, want_labels, want_table, want_stats = CW.components(rows, tri, p)
    out, labels, table, stats = rec.mesh_components(dev(tri), p)
    torch.cuda.synchronize()
    assert CW.stats_dict(stats) == want_stats
    assert np.array_equal(out.cpu().numpy().astype(np.uint32), want_out)
    assert np.array_equal(labels.cpu().numpy(), want_labels)
    assert raw_table(table).tobytes() == want_table.tobytes()
    return want_stats


@pytest.mark.parametrize("name", sorted(HOST.CASES))
def test_bit_equal_on_the_host_cases(name):
    rows, tri = HOST.CASES[name]
    rec = loaded(rows)
    for p in HOST.PARAMS.values():
        assert_same(rec, rows, tri, p)
    rec.close()


def golden_meshes():
    rows = M.golden_f7()
    full = SW.meshed(rows)
    simple, _ = SW.simplify(rows, full, SimplifyParams.defaults())
    return rows, {"full_with_fill": full, "simplified": simple}


@pytest.mark.parametrize("mesh", ["full_with_fill", "simplified"])
def test_bit_equal_on_golden_f7(mesh):
    rows, meshes = golden_meshes()
    rec = loaded(rows)
    for p in HOST.PARAMS.values():
        s = assert_same(rec, rows, meshes[mesh], p)
    assert s["components"] > 1
    rec.close()


@pytest.fixture(scope="module")
def vga():
    """The cloud after the 48-frame VGA stream and its mesh with the fill."""
    rec, st = run_stream(S.Camera.tum(640, 480), 48)
    full = rec.triangulate()[0]
    full = torch.cat([full, rec.fill_holes(full)[0]])
    torch.cuda.synchronize()
    yield rec, st, full
    rec.close()


def test_bit_equal_on_the_vga_stream(vga):
    rec, st, full = vga
    rows, _, _ = rec.dump_state()
    tri = full.cpu().numpy()
    for p in HOST.PARAMS.values():
        s = assert_same(rec, rows, tri, p)
    print(f"VGA stream, {len(tri)} triangles: {s}")
    assert s["components"] > 1


def test_read_only(vga):
    rec, st, full = vga
    before, n, merges = rec.dump_state()
    rec.mesh_components(full, ComponentParams.defaults(keep_largest=3))
    after, n2, merges2 = rec.dump_state()
    assert (n2, merges2) == (n, merges)
    assert np.array_equal(before.view(np.uint32), after.view(np.uint32))


def test_output_feeds_the_other_mesh_calls(vga):
    rec, st, full = vga
    kept, _, _, stats = rec.mesh_components(full)
    assert 0 < len(kept) <= len(full)
    simple, s = rec.simplify_mesh(kept)
    assert s.triangles_in == len(kept) and 0 < len(simple) <= len(kept)
    first, last = st.integrated_range()
    cam = st.camera
    views = [R.TextureView(st.color[f], cam, view_T_global=st.frame_T_global[f], near=0.1, far=20.0)
             for f in range(first, last, 8)]
    atlas, uv, t = rec.texture_mesh(kept, views, TextureParams.defaults(texel_size=0.01))
    assert t.triangles == len(kept) and t.texels_seen > 0
    image = rec.render_mesh(kept, st.frame_T_global[first], cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy,
                            near=0.1, far=20.0, unmeshed_surfels=False, outputs=("depth",))["depth"]
    assert (image > 0).float().mean() > 0.1


def test_labels_and_table_after_compaction():
    rec, st = run_stream(S.Camera.tum(320, 240), 48)
    _, _, merges = rec.dump_state()
    assert merges > 0
    tri = rec.triangulate()[0]
    tri = torch.cat([tri, rec.fill_holes(tri)[0]])
    p = ComponentParams.defaults(min_triangles=5, keep_largest=6)
    out, labels, table, stats = rec.mesh_components(tri, p)
    _, m = rec.compact(return_map=True)
    mapped = R.remap_triangles(tri, m)
    assert len(mapped) == len(tri)
    out2, labels2, table2, stats2 = rec.mesh_components(mapped, p)
    assert CW.stats_dict(stats2) == CW.stats_dict(stats)
    assert torch.equal(labels2, labels) and raw_table(table2).tobytes() == raw_table(table).tobytes()
    assert torch.equal(out2, R.remap_triangles(out, m))
    rec.close()


def test_errors_write_nothing_and_capacity_protocol():
    rows, tri = HOST.CASES["islands"]
    rec = loaded(rows)
    p = ComponentParams.defaults(min_triangles=2)
    want_out, want_labels, want_table, want_stats = CW.components(rows, tri, p)
    fn = rec.lib.fn["mesh_components"]
    src = dev(tri)
    T, P, K = len(tri), len(want_table), len(want_out)
    out = torch.full((T + 1, 3), -7, dtype=torch.int32, device="cuda")
    labels = torch.full((T + 1,), -7, dtype=torch.int32, device="cuda")
    table = torch.full((P + 1, 48), 7, dtype=torch.uint8, device="cuda")
    stats = ComponentStats()

    def ptr(t):
        return C.c_void_p(t.data_ptr()) if t is not None else None

    def call(t=src, params=p, count=None, o=out, oc=None, lab=labels, tab=table, tc=None, st=stats):
        if not isinstance(t, torch.Tensor) and t is not None:
            t = dev(t)
        status = fn(rec._h, None, C.byref(params) if params is not None else None, ptr(t),
                    (len(t) if t is not None else 3) if count is None else count, ptr(o),
                    (len(o) if o is not None else 0) if oc is None else oc, ptr(lab), ptr(tab),
                    (len(tab) if tab is not None else 0) if tc is None else tc, C.byref(st) if st is not None else None)
        torch.cuda.synchronize()
        return status

    def untouched():
        return bool((out == -7).all() and (labels == -7).all() and (table == 7).all())

    launches = rec.lib.fn["kernel_launch_count"]()
    INVALID = _lib.SM_ERR_INVALID_ARGUMENT
    for bad in (ComponentParams.defaults(min_area=-1e-9), ComponentParams.defaults(min_area=float("nan")),
                ComponentParams.defaults(min_area=float("inf"))):
        assert call(params=bad) == INVALID
    assert call(params=None) == INVALID
    assert call(st=None) == INVALID
    assert call(t=None) == INVALID                                   # triangles NULL with a count
    assert call(count=1 << 28) == INVALID
    assert call(o=None, oc=5) == INVALID                             # out NULL with a capacity
    assert call(tab=None, tc=5) == INVALID                           # table NULL with a capacity
    assert call(o=src) == INVALID                                    # out overlaps triangles
    assert call(lab=src.view(-1)) == INVALID                         # labels overlaps triangles
    assert call(tab=src.view(torch.uint8)) == INVALID                # table overlaps triangles
    assert call(lab=out.view(-1)) == INVALID                         # labels overlaps out
    assert call(tab=out.view(torch.uint8).view(-1, 12)) == INVALID   # table overlaps out
    assert call(tab=labels.view(torch.uint8).view(-1, 4)) == INVALID  # table overlaps labels
    assert rec.lib.fn["kernel_launch_count"]() == launches
    assert CW.stats_dict(stats) == dict.fromkeys(CW.STATS, 0) and untouched()
    n = rows.shape[1]
    merged = rows.copy()
    merged[7, 5] = -merged[7, 5]
    # (-1 corners, as int32 padding or SM_INVALID_SURFEL_INDEX, give an undirected edge key equal to the edge table's
    # empty key)
    for t in (np.concatenate([tri, [[0, 1, n]]]), np.concatenate([tri, [[0, 0, 1]]]),
              np.concatenate([tri, [[0, -1, -1]]]), np.concatenate([[[-1, -1, -1]], tri]),
              np.concatenate([tri[:3], [[-1, 2, -1]], tri[3:]])):
        assert call(t) == INVALID
        assert CW.stats_dict(stats) == dict.fromkeys(CW.STATS, 0) and untouched()
    assert rec.lib.fn["last_error"]() == b"sm_mesh_components: a corner is not a present slot below surfels_size()"
    # a count query, out and table one short, then enough
    assert call(o=None, lab=None, tab=None) == _lib.SM_ERR_CAPACITY and CW.stats_dict(stats) == want_stats
    assert call(oc=K - 1) == _lib.SM_ERR_CAPACITY and CW.stats_dict(stats) == want_stats
    assert rec.lib.fn["last_error"]() == f"sm_mesh_components: {K} triangles do not fit the capacity of {K - 1}".encode()
    assert call(tc=P - 1) == _lib.SM_ERR_CAPACITY and CW.stats_dict(stats) == want_stats
    assert rec.lib.fn["last_error"]() == f"sm_mesh_components: {P} pieces do not fit the table capacity of {P - 1}".encode()
    assert untouched()
    assert call(oc=K, tc=P) == _lib.SM_OK and CW.stats_dict(stats) == want_stats
    assert np.array_equal(out[:K].cpu().numpy().astype(np.uint32), want_out) and (out[K:] == -7).all()
    assert np.array_equal(labels[:T].cpu().numpy(), want_labels) and (labels[T:] == -7).all()
    assert table[:P].cpu().numpy().tobytes() == want_table.tobytes() and (table[P:] == 7).all()
    assert call(lab=None, tab=None, tc=0) == _lib.SM_OK                # labels and table may be NULL
    assert call(np.zeros((0, 3)), o=None, lab=None, tab=None) == _lib.SM_OK and stats.components == 0
    rec2 = loaded(merged)                                               # a merged slot is not present
    stats2 = ComponentStats()
    before = out.clone()
    assert rec2.lib.fn["mesh_components"](rec2._h, None, C.byref(p), ptr(src), T, ptr(out), T + 1, None, None, 0,
                                          C.byref(stats2)) == INVALID
    torch.cuda.synchronize()
    assert CW.stats_dict(stats2) == dict.fromkeys(CW.STATS, 0) and torch.equal(out, before)
    rec2.close()
    rec.close()


def test_obj_export(tmp_path):
    rec, st = run_stream(S.Camera.tum(320, 240), 16, stream_id=3)
    p = ComponentParams.defaults()
    holes = HoleParams.defaults()
    rec.save_mesh_obj(tmp_path / "plain.obj", holes=holes)
    rec.save_mesh_obj(tmp_path / "kept.obj", holes=holes, components=p)
    tri, _ = rec.triangulate()
    tri = torch.cat([tri, rec.fill_holes(tri, holes)[0]])
    kept, _, _, stats = rec.mesh_components(tri, p)
    assert stats.components > 1
    v0, _, f0 = mesh_io.read_obj(tmp_path / "plain.obj")
    v, _, f = mesh_io.read_obj(tmp_path / "kept.obj")
    assert len(f) == len(kept) and len(v) == len(np.unique(kept.cpu().numpy()))
    # the same faces as the kept triangles, over only the slots they use
    positions, _ = rec.export_vertices_host()
    assert np.allclose(v[f], positions[kept.cpu().numpy()], atol=1e-5)
    rec.close()
