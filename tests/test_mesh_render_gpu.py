"""sm_render_mesh on the GPU: bit-exact against the plain-C restatement (tests/mesh_render_walk.c) on hand-built
meshes, the golden state and integrated synthetic streams (with and without the disks of unmeshed surfels), at
sizes from 1x1 to 1280x960; the empty list against sm_render_surfels; output layouts, argument checks, read-only
behaviour, sessions, and the rendered depth against the analytic scene the stream was ray-cast from."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import RenderParams
from tests import mesh_render_walk as MRW
from tests import mesh_walk as M
from tests.test_mesh_render_host import CAM as GRID_CAM, fan, grid_mesh, vertex_rows
from tests.test_render_gpu import (BEHIND, CAM, FAR, IDENTITY, NEAR, OUTPUT_CAMERAS, VGA, ODD, assert_bit_equal, make,
                                   orbit_pose, params)

pytestmark = pytest.mark.gpu

CAMERAS = dict(OUTPUT_CAMERAS, pixel_grid=GRID_CAM)


def walk(rows, tris, T, cam, near=NEAR, far=FAR, disks=True):
    return MRW.render(rows, tris, T, cam["width"], cam["height"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], near,
                      far, unmeshed_surfels=disks)


def gpu(rec, tris, T, cam, near=NEAR, far=FAR, disks=True, outputs=R.RENDER_OUTPUTS):
    t = torch.as_tensor(np.asarray(tris, np.int64).reshape(-1, 3).astype(np.int32), device="cuda") \
        if not isinstance(tris, torch.Tensor) else tris
    out = rec.render_mesh(t, T, near=near, far=far, unmeshed_surfels=disks, outputs=outputs, **cam)
    torch.cuda.synchronize()
    return out


def check(rec, rows, tris, T, cam, near=NEAR, far=FAR, disks=True):
    ref = walk(rows, tris if not isinstance(tris, torch.Tensor) else tris.cpu().numpy(), T, cam, near, far, disks)
    out = gpu(rec, tris, T, cam, near, far, disks)
    assert_bit_equal({k: v.view(torch.int32) if k == "index" else v for k, v in out.items()}, ref)
    return ref


def _grid(diagonal, step, origin, z=1.0):
    pts, tris, _ = grid_mesh(17, 14, step, origin, diagonal, z)
    return pts, tris


def hand_built():
    """name -> (points or rows, triangles); coordinates chosen for the pixel-grid camera, seen by all cameras."""
    cases = {}
    pts, tris = _grid("alternate", 5, (3, 4))
    cases["grid_on_pixel_centres"] = (vertex_rows(pts), tris)
    pts, tris = _grid("/", 3.7, (2.3, 1.9), z=1.7)
    cases["grid_off_centre"] = (vertex_rows(pts), tris[:, ::-1])
    rng = np.random.default_rng(5)
    ring = fan(rng, 11, np.array([48.0, 40.0]), jitter=True)
    z = rng.uniform(0.8, 2.5, 12)
    scr = np.vstack([[48.0, 40.0], ring])
    pts = [((u - 0.5) / 64.0 * zz, (v - 0.5) / 64.0 * zz, zz) for (u, v), zz in zip(scr, z)]
    cases["random_fan"] = (vertex_rows(pts), np.array([(0, 1 + i, 1 + (i + 1) % 11) for i in range(11)]))
    # disks of non-corner slots in the plane of the grid: exact depth ties at the vertex pixels, triangles win
    pts, tris = _grid("\\", 5, (3, 4))
    rows = vertex_rows(pts + [((3 + 5 * i) / 64.0, (4 + 5 * j) / 64.0, 1.0) for i in range(16) for j in range(13)])
    rows[7, len(pts):] = (4.0 / 64.0) ** 2
    cases["ties_with_disks"] = (rows, tris)
    # corners crossing the near plane, beyond far, merged corners and stale indices
    pts = [(-0.2, -0.2, 1.0), (0.3, -0.2, 1.0), (0.0, 0.3, 1.0), (0.1, 0.1, 0.05), (0.2, 0.0, 30.0), (0.25, 0.25, 1.2),
           (-0.25, 0.2, 1.1)]
    rows = vertex_rows(pts)
    rows[7, 6] = -rows[7, 6]
    cases["near_far_merged_stale"] = (rows, np.array([(0, 1, 3), (0, 1, 4), (0, 2, 6), (1, 2, 5), (0, 5, 99),
                                                      (7, 1, 2), (0, 1, 2)]))
    # one triangle around the whole view, and many large ones
    rows = vertex_rows([(-40.0, -40.0, 2.0), (40.0, -40.0, 2.5), (0.0, 60.0, 3.0)])
    cases["whole_image"] = (rows, np.array([(0, 1, 2)]))
    pts, tris = _grid("alternate", 24, (-20, -25), z=0.6)
    cases["many_large"] = (vertex_rows(pts), tris)
    cases["empty"] = (vertex_rows([(0.0, 0.0, 1.0), (0.1, 0.0, 1.2)]), np.zeros((0, 3), np.int64))
    return cases


HAND_BUILT = hand_built()


@pytest.mark.parametrize("disks", [True, False], ids=["with_disks", "triangles_only"])
@pytest.mark.parametrize("case", sorted(HAND_BUILT))
@pytest.mark.parametrize("cam", sorted(CAMERAS))
def test_hand_built_meshes_bit_exact(case, cam, disks):
    rows, tris = HAND_BUILT[case]
    rec = make()
    rec.load_state(rows, 0)
    T = IDENTITY.copy()
    if cam != "pixel_grid":
        T[:, 3] = (-0.55, -0.45, 0.8)   # the pixel-grid scenes sit right of and below the axis: move them in front
    ref = check(rec, rows, tris, T, CAMERAS[cam], disks=disks)
    if case not in ("empty",):
        assert (ref["index"] != MRW.INVALID).sum() > 0
    if case == "whole_image" and cam == "pixel_grid":
        assert np.all(ref["index"] == 0)
    if case == "ties_with_disks" and cam == "pixel_grid" and disks:
        tri = ref["index"] < MRW.DISK
        assert tri.sum() > 1000 and (ref["index"] == MRW.INVALID).sum() < ref["index"].size


def test_golden_state_with_its_mesh():
    from tests.util import GOLDEN_DIR
    meta = np.load(GOLDEN_DIR / "golden_320x240_meta.npz")
    w, h, fx, fy, cx, cy = [float(v) for v in meta["camera"]]
    cam = dict(width=int(w), height=int(h), fx=fx, fy=fy, cx=cx, cy=cy)
    rows = M.golden_f7()
    rec = make()
    rec.load_state(rows, 0)
    tris, stats = rec.triangulate()
    want, _, _ = M.triangulate(rows)
    assert np.array_equal(tris.cpu().numpy().astype(np.uint32), want)
    for T in (meta["frame_T_global"][7], meta["frame_T_global"][4]):
        for disks in (True, False):
            ref = check(rec, rows, tris, T, cam, near=0.1, far=100.0, disks=disks)
            assert ((ref["index"] != MRW.INVALID) & (ref["index"] < MRW.DISK)).mean() > 0.1


@pytest.fixture(scope="module")
def integrated():
    """The cloud after 40 integrated frames of the VGA synthetic stream and its sm_triangulate mesh."""
    st = S.make_stream(CAM, 48, device="cuda")
    pp, ip = params()
    rec = make()
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    rows, n, _ = rec.dump_state()
    tris, _ = rec.triangulate()
    torch.cuda.synchronize()
    return st, rec, rows.copy(), n, tris


POSES = {"input": lambda st: st.frame_T_global[30], "orbit": lambda st: orbit_pose(st, 30, 35.0, 0.4),
         "behind": lambda st: BEHIND}


@pytest.mark.parametrize("disks", [True, False], ids=["with_disks", "triangles_only"])
@pytest.mark.parametrize("pose", sorted(POSES))
@pytest.mark.parametrize("cam", ["vga", "odd", "negative_fy"])
def test_integrated_mesh_bit_exact(integrated, pose, cam, disks):
    st, rec, rows, n, tris = integrated
    T = POSES[pose](st)
    ref = check(rec, rows, tris, T, OUTPUT_CAMERAS[cam], disks=disks)
    assert (ref["index"] != MRW.INVALID).mean() > 0.2
    again = gpu(rec, tris, T, OUTPUT_CAMERAS[cam], disks=disks)      # the key raster and list counts are restored
    assert_bit_equal({k: v.view(torch.int32) if k == "index" else v for k, v in again.items()}, ref)


def test_large_image_and_tiny_images(integrated):
    st, rec, rows, n, tris = integrated
    big = dict(width=1280, height=960, fx=2 * CAM.fx, fy=2 * CAM.fy, cx=2 * CAM.cx, cy=2 * CAM.cy)
    T = orbit_pose(st, 20, -25.0, 0.2)
    check(rec, rows, tris, T, big)
    for w, h in ((1, 1), (2, 1)):
        cam = dict(width=w, height=h, fx=0.5, fy=0.5, cx=w / 2, cy=h / 2)
        check(rec, rows, tris, st.frame_T_global[30], cam)


def test_empty_list_with_the_flag_is_render_surfels(integrated):
    st, rec, rows, n, tris = integrated
    T = st.frame_T_global[25]
    empty = torch.zeros((0, 3), dtype=torch.int32, device="cuda")
    disks = gpu(rec, empty, T, VGA)
    plain = rec.render(T, near=NEAR, far=FAR, **VGA)
    torch.cuda.synchronize()
    for k in ("depth", "color", "normal"):
        assert torch.equal(disks[k].view(torch.uint8), plain[k].view(torch.uint8)), k
    valid = plain["index"] >= 0
    assert valid.float().mean() > 0.2
    assert torch.equal(disks["index"][valid], plain["index"][valid] | np.int32(-2**31))
    assert torch.equal(disks["index"][~valid], plain["index"][~valid])
    check(rec, rows, empty, T, VGA)
    none = gpu(rec, empty, T, VGA, disks=False)
    assert bool((none["index"] == -1).all()) and bool((none["depth"] == 0).all())


def raw(rec, tris, count, flags, T, cam, bufs, near=NEAR, far=FAR):
    """sm_render_mesh through the C ABI; bufs: name -> tensor (None = NULL) or (pointer, pitch)."""
    args = []
    for k in R.RENDER_OUTPUTS:
        b = bufs.get(k)
        if b is None:
            args += [None, 0]
        elif isinstance(b, tuple):
            args += [C.c_void_p(b[0]), b[1]]
        else:
            args += [C.c_void_p(b.data_ptr()), b.stride(0) * b.element_size()]
    p = RenderParams(cam["width"], cam["height"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], near, far)
    T = np.ascontiguousarray(np.asarray(T, np.float32).reshape(-1)[:12])
    ptr = C.c_void_p(tris.data_ptr()) if tris is not None else None
    return rec.lib.fn["render_mesh"](rec._h, torch.cuda.current_stream().cuda_stream, C.byref(p),
                                     T.ctypes.data_as(C.c_void_p), ptr, count, flags, *args)


def test_pitched_outputs_and_subsets(integrated):
    st, rec, rows, n, tris = integrated
    T = st.frame_T_global[25]
    H, W = ODD["height"], ODD["width"]
    pad = 7
    bufs = {"depth": torch.full((H, W + pad), -3.5, dtype=torch.float32, device="cuda"),
            "color": torch.full((H, W + pad, 3), 0xAB, dtype=torch.uint8, device="cuda"),
            "normal": torch.full((H, W + pad, 3), 9.25, dtype=torch.float32, device="cuda"),
            "index": torch.full((H, W + pad), 0x5A5A5A5A, dtype=torch.int32, device="cuda")}
    before = {k: v.clone() for k, v in bufs.items()}
    assert raw(rec, tris, tris.shape[0], 1, T, ODD, bufs) == _lib.SM_OK
    torch.cuda.synchronize()
    ref = walk(rows, tris.cpu().numpy(), T, ODD)
    assert_bit_equal({k: v[:, :W] for k, v in bufs.items()}, ref)
    for k in bufs:
        assert torch.equal(bufs[k][:, W:], before[k][:, W:]), k
    for k in R.RENDER_OUTPUTS:
        out = gpu(rec, tris, T, ODD, outputs=(k,))
        assert set(out) == {k}
        assert_bit_equal(out, ref, (k,))


def test_render_mesh_only_reads_the_state_and_repeats():
    st = S.make_stream(CAM, 24, device="cuda")
    pp, ip = params()
    rec = make()
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    rec.mesh_update()
    tris = rec.mesh_triangles("all")
    before, n0, m0 = rec.dump_state()
    before = before.copy()
    a = gpu(rec, tris, st.frame_T_global[15], VGA)
    b = gpu(rec, tris, st.frame_T_global[15], VGA)
    gpu(rec, tris, BEHIND, VGA, disks=False)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    after, n1, m1 = rec.dump_state()
    assert (n0, m0) == (n1, m1)
    assert np.array_equal(before.view(np.uint32), after.view(np.uint32))
    assert rec.mesh_update().slots_changed == 0


def test_render_mesh_between_session_pushes():
    st = S.make_stream(CAM, 40, device="cuda")
    pp, ip = params()
    rec = make()
    seen = []
    with rec.session(pp, ip, (CAM.width, CAM.height)) as s:
        for f in range(st.frame_count):
            status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            if f not in (20, 33):
                continue
            rec.mesh_update()
            tris = rec.mesh_triangles("all")
            T = st.frame_T_global[int(status.last_integrated_frame)]
            out = gpu(rec, tris, T, VGA)
            rows, n, merges = rec.dump_state()
            ref = walk(rows, tris.cpu().numpy(), T, VGA)
            assert_bit_equal({k: v.view(torch.int32) if k == "index" else v for k, v in out.items()}, ref)
            assert ((ref["index"] != MRW.INVALID) & (ref["index"] < MRW.DISK)).mean() > 0.1
            seen.append(f)
    assert seen == [20, 33]


def test_invalid_arguments_are_rejected_without_a_launch(integrated, product):
    st, rec, rows, n, tris = integrated
    H, W = 8, 10
    ok = {"depth": torch.zeros((H, W), dtype=torch.float32, device="cuda")}
    cam = dict(width=W, height=H, fx=10.0, fy=10.0, cx=5.0, cy=4.0)
    T = IDENTITY
    count = tris.shape[0]
    assert raw(rec, tris, count, 1, T, cam, ok) == _lib.SM_OK
    torch.cuda.synchronize()
    nan, inf = float("nan"), float("inf")
    launches = product.fn["kernel_launch_count"]()
    bad_cams = [dict(cam, width=0), dict(cam, height=-1), dict(cam, fx=0.0), dict(cam, fy=nan), dict(cam, fx=inf),
                dict(cam, cx=nan), dict(cam, cy=inf)]
    for c in bad_cams:
        assert raw(rec, tris, count, 1, T, c, ok) == _lib.SM_ERR_INVALID_ARGUMENT, c
    for near, far in [(0.0, 1.0), (-1.0, 1.0), (1.0, 1.0), (2.0, 1.0), (nan, 1.0), (0.1, nan)]:
        assert raw(rec, tris, count, 1, T, cam, ok, near, far) == _lib.SM_ERR_INVALID_ARGUMENT, (near, far)
    for k in range(12):
        Tb = IDENTITY.copy().reshape(-1)
        Tb[k] = nan if k % 2 else inf
        assert raw(rec, tris, count, 1, Tb, cam, ok) == _lib.SM_ERR_INVALID_ARGUMENT, k
    assert raw(rec, tris, count, 1, T, cam, {}) == _lib.SM_ERR_INVALID_ARGUMENT
    big = torch.zeros(H * W * 16, dtype=torch.uint8, device="cuda")
    for k, row in {"depth": 4 * W, "color": 3 * W, "normal": 12 * W, "index": 4 * W}.items():
        assert raw(rec, tris, count, 1, T, cam, {k: (big.data_ptr(), row - 1)}) == _lib.SM_ERR_INVALID_ARGUMENT, k
    assert raw(rec, None, 5, 1, T, cam, ok) == _lib.SM_ERR_INVALID_ARGUMENT
    assert raw(rec, tris, 2**31, 1, T, cam, ok) == _lib.SM_ERR_INVALID_ARGUMENT
    for flags in (2, -1, 0x100, 1 | 4):
        assert raw(rec, tris, count, flags, T, cam, ok) == _lib.SM_ERR_INVALID_ARGUMENT, flags
    assert rec.lib.fn["render_mesh"](rec._h, None, None, T.ctypes.data_as(C.c_void_p), None, 0, 0,
                                     *([None, 0] * 4)) == _lib.SM_ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert product.fn["kernel_launch_count"]() == launches
    assert raw(rec, None, 0, 0, T, cam, ok) == _lib.SM_OK            # an empty list is legal
    assert raw(rec, tris, count, 0, T, cam, ok) == _lib.SM_OK
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        rec.render_mesh(tris.long(), T, **cam)


# Rendered from the input pose of frame 40 after frames 4..43 of the 48-frame VGA stream, with sm_triangulate's mesh
# and the disks of the unmeshed surfels, against the float64 ray cast of that pose. Measured on an H100 80GB HBM3
# (700 W power limit):
#   nominal noise: median |d| 0.62 mm, p95 4.46 mm, coverage 0.478 (0.478 by triangles)
#   noise free:    median |d| 0.58 mm, p95 4.61 mm, coverage 0.481 (0.481 by triangles)
# sm_render_surfels on the same view: 0.71 / 0.62 mm, 5.15 mm, 0.52 (test_render_gpu.py). The mesh leaves holes
# where the disks overlap, so it covers a little less. Limits: twice the measured median, 1.5 times the p95, coverage
# 0.03 below.
SCENE_LIMITS = {
    None: dict(median=0.00125, p95=0.0067, coverage=0.448),
    0.0: dict(median=0.00116, p95=0.0069, coverage=0.451),
}


@pytest.mark.parametrize("sigma", [None, 0.0], ids=["nominal_noise", "noise_free"])
def test_rendered_mesh_depth_matches_the_scene(sigma):
    st = S.make_stream(CAM, 48, sigma_depth=sigma, device="cuda")
    pp, ip = params()
    rec = make()
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    tris, _ = rec.triangulate()
    f = last - 4
    pose64 = torch.from_numpy(S.trajectory(st.frame_count)[f]).to("cuda")
    gt, _ = S._raycast(CAM, pose64, "cuda")
    out = rec.render_mesh(tris, st.frame_T_global[f], near=NEAR, far=FAR, outputs=("depth", "index"), **VGA)
    depth = out["depth"].double()
    gt_valid = torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0)
    both = gt_valid & (depth > 0)
    err = (depth - gt)[both].abs().cpu().numpy()
    median, p95 = float(np.median(err)), float(np.percentile(err, 95))
    coverage = float(both.sum()) / float(gt_valid.sum())
    tri = (gt_valid & (out["index"] >= 0)).sum().item() / float(gt_valid.sum())
    print(f"mesh scene sigma={sigma}: median |d| {median:.6f} m, p95 {p95:.6f} m, coverage {coverage:.5f} "
          f"(triangles {tri:.5f})")
    lim = SCENE_LIMITS[sigma]
    assert median <= lim["median"] and p95 <= lim["p95"] and coverage >= lim["coverage"]
