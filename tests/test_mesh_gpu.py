"""sm_triangulate on the GPU: bit-exact against the plain-C restatement (tests/mesh_walk.c) on hand-built clouds,
the golden f7 state and integrated synthetic streams; repeatability, read-only behaviour, the capacity error,
argument checks, sessions, distance to the analytic scene and, where the reference's CPU mesher is built, its
triangle count and area on the same cloud."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, MeshParams, MeshStats, PreprocessParams
from tests import mesh_walk as M

pytestmark = pytest.mark.gpu

CAP = 2_000_000


def make(cam, cap=CAP):
    return R.CUDASurfelReconstruction(cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


def loaded(rows):
    rec = make(S.Camera.tum(320, 240), cap=max(rows.shape[1], 1024))
    rec.load_state(rows, 0)
    return rec


def gpu_mesh(rec, params=None):
    tri, stats = rec.triangulate(params)
    torch.cuda.synchronize()
    return tri.cpu().numpy().astype(np.uint32), {k: int(getattr(stats, k)) for k, _ in MeshStats._fields_}


def assert_same(rows, got, params=None):
    want_tri, want_stats, _ = M.triangulate(rows, params)
    tri, stats = got
    assert stats == want_stats
    assert tri.shape == want_tri.shape
    bad = np.flatnonzero((tri != want_tri).any(1))
    assert bad.size == 0, f"{bad.size} differing triangles, first #{bad[:1]}: {tri[bad[:1]]} vs {want_tri[bad[:1]]}"


def run_stream(cam, frames, stream_id=0):
    st = S.make_stream(cam, frames, stream_id=stream_id, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    rec = make(cam)
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                   IntegrateParams.defaults(), first, last)
    return rec, st


@pytest.mark.parametrize("name", sorted(M.CASES) + ["golden_f7"])
def test_bit_equal_to_restatement(name):
    rows = M.golden_f7() if name == "golden_f7" else M.CASES[name]()
    rec = loaded(rows)
    got = gpu_mesh(rec)
    M.check_invariants(rows, got[0])
    assert_same(rows, got)
    # other parameters: a tighter normal gate and triangle angle, a larger search radius
    p = MeshParams(2.5, 40.0, 120.0)
    assert_same(rows, gpu_mesh(rec, p), p)
    rec.close()


# (the first and last K/2 = 4 frames of a stream are not integrated)
@pytest.mark.parametrize("size,frames", [((320, 240), 16), ((640, 480), 12)])
def test_bit_equal_on_integrated_streams(size, frames):
    rec, _ = run_stream(S.Camera.tum(*size), frames, stream_id=3)
    rows, n, _ = rec.dump_state()
    got = gpu_mesh(rec)
    assert got[1]["triangle_count"] > n // 2
    M.check_invariants(rows, got[0])
    assert_same(rows, got)
    rec.close()


def test_repeatable_and_read_only():
    rec = loaded(M.golden_f7())
    before, _, _ = rec.dump_state()
    a = gpu_mesh(rec)
    b = gpu_mesh(rec)
    after, _, _ = rec.dump_state()
    assert a[1] == b[1] and np.array_equal(a[0], b[0])
    assert np.array_equal(before.view(np.uint32), after.view(np.uint32))
    rec.close()


def test_capacity_error_writes_nothing():
    rec = loaded(M.jittered_plane())
    want = gpu_mesh(rec)[1]["triangle_count"]
    buf = torch.full((want - 1, 3), -7, dtype=torch.int32, device="cuda")
    stats = MeshStats()
    p = MeshParams.defaults()
    status = rec.lib.fn["triangulate"](rec._h, None, C.byref(p), C.c_void_p(buf.data_ptr()), want - 1, C.byref(stats))
    torch.cuda.synchronize()
    assert status == _lib.SM_ERR_CAPACITY
    assert stats.triangle_count == want and stats.vertices_meshed > 0
    assert (buf == -7).all()
    rec.close()


def test_invalid_arguments_launch_nothing():
    rec = loaded(M.jittered_plane())
    stats = MeshStats()
    buf = torch.zeros((10, 3), dtype=torch.int32, device="cuda")
    fn = rec.lib.fn["triangulate"]
    bad = [MeshParams(0.0, 90, 170), MeshParams(-1.0, 90, 170), MeshParams(math.nan, 90, 170),
           MeshParams(math.inf, 90, 170), MeshParams(2, 0.0, 170), MeshParams(2, 180.5, 170),
           MeshParams(2, 90, 0.0), MeshParams(2, 90, math.nan), MeshParams(2, 90, 200)]
    launches = rec.lib.fn["kernel_launch_count"]()
    for p in bad:
        assert fn(rec._h, None, C.byref(p), C.c_void_p(buf.data_ptr()), 10, C.byref(stats)) == _lib.SM_ERR_INVALID_ARGUMENT
    p = MeshParams.defaults()
    assert fn(rec._h, None, None, C.c_void_p(buf.data_ptr()), 10, C.byref(stats)) == _lib.SM_ERR_INVALID_ARGUMENT
    assert fn(rec._h, None, C.byref(p), C.c_void_p(buf.data_ptr()), 10, None) == _lib.SM_ERR_INVALID_ARGUMENT
    assert fn(rec._h, None, C.byref(p), None, 10, C.byref(stats)) == _lib.SM_ERR_INVALID_ARGUMENT
    assert rec.lib.fn["kernel_launch_count"]() == launches
    # a count query: NULL buffer, capacity 0
    assert fn(rec._h, None, C.byref(p), None, 0, C.byref(stats)) == _lib.SM_ERR_CAPACITY
    assert stats.triangle_count == gpu_mesh(rec)[1]["triangle_count"]
    rec.close()


def test_triangulate_between_session_pushes():
    cam = S.Camera.tum(320, 240)
    st = S.make_stream(cam, 24, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    rec = make(cam)
    seen = []
    with rec.session(pp, IntegrateParams.defaults(), (cam.width, cam.height)) as s:
        for f in range(st.frame_count):
            status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            if f not in (12, 19):
                continue
            got = gpu_mesh(rec)
            rows, n, merges = rec.dump_state()
            other = loaded(rows)
            assert gpu_mesh(other)[1] == got[1]
            assert_same(rows, got)
            other.close()
            seen.append(int(status.last_integrated_frame))
    assert len(seen) == 2 and seen[0] < seen[1]
    rec.close()


def scene_distance(points):
    """Unsigned distance (float64) from points to the analytic scene of surfelmeshing_b200.synthetic: the floor
    z = 0, the walls |x| = |y| = _ROOM and every _SCENE box and sphere."""
    p = np.asarray(points, np.float64)
    best = np.abs(p[:, 2])
    best = np.minimum(best, np.abs(np.abs(p[:, 0]) - S._ROOM))
    best = np.minimum(best, np.abs(np.abs(p[:, 1]) - S._ROOM))
    for kind, prm, _ in S._SCENE:
        if kind == "sphere":
            c, r = np.asarray(prm[0], np.float64), float(prm[1])
            best = np.minimum(best, np.abs(np.linalg.norm(p - c, axis=1) - r))
        else:
            lo, hi = np.asarray(prm[0], np.float64), np.asarray(prm[1], np.float64)
            q = np.abs(p - (lo + hi) / 2) - (hi - lo) / 2
            outside = np.linalg.norm(np.maximum(q, 0), axis=1)
            best = np.minimum(best, np.abs(outside + np.minimum(q.max(1), 0)))
    return best


# Triangle centroids of the 48-frame VGA stream against the analytic scene. Measured on an H100 80GB HBM3 (700 W
# power limit): 267 745 triangles, median 0.365 mm, p95 2.11 mm. Limits: about twice the median, 1.5 times the p95.
SCENE_MEDIAN_M = 0.0008
SCENE_P95_M = 0.0032


def test_centroids_lie_on_the_scene():
    rec, _ = run_stream(S.Camera.tum(640, 480), 48)
    tri, stats = gpu_mesh(rec)
    rows, n, _ = rec.dump_state()
    p = rows[3:6].T.astype(np.float64)
    centroids = p[tri.astype(np.int64)].mean(1)
    d = scene_distance(centroids)
    med, p95 = float(np.median(d)), float(np.percentile(d, 95))
    print(f"scene distance: median {med * 1e3:.3f} mm, p95 {p95 * 1e3:.3f} mm, {len(tri)} triangles, {stats}")
    assert med < SCENE_MEDIAN_M and p95 < SCENE_P95_M
    rec.close()


def test_against_reference_cpu_mesher():
    from oracle import meshing_ref
    if not meshing_ref.available():
        pytest.skip("oracle/_ref/libmeshing_ref.so not built")
    rows = M.golden_f7()
    rec = loaded(rows)
    tri, _ = gpu_mesh(rec)
    ref = meshing_ref.SurfelMeshing()
    keep = rows[7] > 0
    ref.integrate(1, *[rows[k] for k in (3, 4, 5, 7, 8, 9, 10)], rows[18].view(np.uint32))
    ref.check_remeshing()
    ref.triangulate()
    rt = ref.triangles()
    ref.close()
    ratio_count = len(tri) / max(len(rt), 1)
    ratio_area = M.area(rows, tri) / max(M.area(rows, rt), 1e-12)
    print(f"reference CPU mesher: {len(rt)} triangles; this: {len(tri)} ({ratio_count:.3f}, area {ratio_area:.3f})")
    # Calibrated on the CPU with the restatement (which the GPU matches bit for bit): 21 217 triangles against the
    # reference's 21 562 (0.984), area 0.931 of the reference's.
    assert 0.90 < ratio_count < 1.08 and 0.85 < ratio_area < 1.05
    assert keep.any()
    rec.close()
