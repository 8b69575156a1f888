"""sm_render_surfels on the GPU: bit-exact against the plain-C restatement (tests/render_walk.c) on hand-built clouds
and on integrated synthetic streams, output layouts, argument checks, read-only behaviour, sessions, and the rendered
depth against the analytic scene the stream was ray-cast from."""
import ctypes as C

import numpy as np
import pytest
import torch

from surfelmeshing_b200 import _lib, synthetic as S
from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, RenderParams
from tests import render_walk
from tests.test_render_host import make_rows

pytestmark = pytest.mark.gpu

CAM = S.Camera.tum(640, 480)
CAP = 2_000_000
NEAR, FAR = 0.1, 20.0
IDENTITY = np.eye(4, dtype=np.float32)[:3]
# an output camera unlike the handle's: non-square, odd sizes, fx != fy, off-centre principal point
ODD = dict(width=333, height=197, fx=300.0, fy=310.0, cx=170.3, cy=95.6)
VGA = dict(width=CAM.width, height=CAM.height, fx=CAM.fx, fy=CAM.fy, cx=CAM.cx, cy=CAM.cy)
# an ICL-NUIM-like output camera: negative fy (the image is flipped vertically; axis_range swaps the bounds for f < 0)
FLIPPED = dict(width=CAM.width, height=CAM.height, fx=481.2, fy=-480.0, cx=320.0, cy=240.0)
OUTPUT_CAMERAS = {"vga": VGA, "odd": ODD, "negative_fy": FLIPPED}


def make(lib=None):
    return R.CUDASurfelReconstruction(CAP, CAM.width, CAM.height, CAM.fx, CAM.fy, CAM.cx, CAM.cy, lib=lib)


def params(cam=CAM):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    return pp, IntegrateParams.defaults()


def walk(rows, T, near=NEAR, far=FAR, **cam):
    return render_walk.render(rows, T, cam["width"], cam["height"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], near,
                              far)


def assert_bit_equal(out, ref, outputs=R.RENDER_OUTPUTS):
    for k in outputs:
        got = out[k].cpu().numpy()
        want = ref[k]
        if got.dtype != np.uint8:
            got, want = got.view(np.uint32), want.view(np.uint32)
        bad = got != want
        assert not bad.any(), f"{k}: {int(bad.sum())} differing values, first at {np.argwhere(bad)[0].tolist()}"


def view_from(global_T_camera):
    return R.invert_rigid(np.asarray(global_T_camera, np.float64))


def orbit_pose(st, frame, degrees, lift):
    """An off-trajectory camera: the eye of `frame` turned about the world z axis and raised, looking at the desk."""
    eye = np.asarray(st.global_T_frame[frame], np.float64)[:, 3]
    a = np.radians(degrees)
    rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    return view_from(S._look_at(rz @ eye + np.array([0, 0, lift]), np.array([0.0, 0.0, 0.8])))


BEHIND = view_from(S._look_at(np.array([0.5, -0.4, -1.2]), np.array([0.0, 0.0, 0.5])))   # under the floor, looking up

HAND_BUILT = {
    "single": [((0.05, -0.03, 2.0), (0, 0, -1), 0.2, (10, 20, 30))],
    "tilted": [((-0.3, 0.1, 1.5), (0.6, -0.2, -0.75), 0.25, (1, 2, 3))],
    "overlapping": [((0.0, 0.0, 2.0), (0, 0, -1), 0.3, (50, 0, 0)), ((0.1, 0.05, 1.8), (0.2, 0, -1), 0.2, (0, 50, 0)),
                    ((-0.1, 0.0, 2.2), (0, 0.3, -1), 0.4, (0, 0, 50))],
    "equal_depth": [((0.0, 0.0, 2.0), (0, 0, -1), 0.3, (50, 0, 0)), ((0.0, 0.0, 2.0), (0, 0, -1), 0.3, (0, 50, 0)),
                    ((0.05, 0.0, 2.0), (0, 0, -1), 0.3, (0, 0, 50))],
    "merged": [((0.0, 0.0, 2.0), (0, 0, -1), -0.5, (9, 9, 9)), ((0.0, 0.0, 2.0), (0, 0, -1), 0.2, (1, 1, 1))],
    "behind_and_out_of_range": [((0.0, 0.0, -2.0), (0, 0, 1), 0.5, (1, 0, 0)), ((0.0, 0.0, 0.05), (0, 0, -1), 0.01, (2, 0, 0)),
                                ((0.0, 0.0, 25.0), (0, 0, -1), 3.0, (3, 0, 0)), ((0.2, 0.1, 3.0), (0, 0, -1), 0.1, (4, 0, 0))],
    # bounding sphere through the camera plane: the whole image goes to the large-splat pass
    "whole_image": [((0.0, 0.0, 0.3), (0.1, 0.2, -1), 2.0, (5, 6, 7)), ((0.0, 0.0, 0.25), (0, 0, -1), 0.05, (8, 8, 8))],
    # many splats of a few hundred pixels each: the large pass with a long list
    "many_large": [((x, y, 1.0), (0, 0, -1), 0.03, (int(40 * x + 100), int(40 * y + 100), 9))
                   for x in np.linspace(-0.5, 0.5, 12) for y in np.linspace(-0.4, 0.4, 9)],
    "empty": [],
}


@pytest.mark.parametrize("case", sorted(HAND_BUILT))
@pytest.mark.parametrize("cam", ["vga", "odd", "negative_fy"])
def test_hand_built_clouds_bit_exact(case, cam):
    cam = OUTPUT_CAMERAS[cam]
    rows = make_rows(HAND_BUILT[case])
    rec = make()
    rec.load_state(rows, 0)
    out = rec.render(IDENTITY, near=NEAR, far=FAR, **cam)
    torch.cuda.synchronize()
    ref = walk(rows, IDENTITY, **cam)
    assert_bit_equal(out, ref)
    if case not in ("empty", "behind_and_out_of_range"):
        assert (ref["index"] != 0xFFFFFFFF).sum() > 0
    if case == "behind_and_out_of_range":
        assert set(np.unique(ref["index"]).tolist()) <= {3, 0xFFFFFFFF}
    if case == "whole_image":
        assert np.all(ref["index"] != 0xFFFFFFFF)


@pytest.fixture(scope="module")
def integrated():
    """The cloud after 40 integrated frames of the VGA synthetic stream."""
    st = S.make_stream(CAM, 48, device="cuda")
    pp, ip = params()
    rec = make()
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    rows, n, _ = rec.dump_state()
    return st, rec, rows.copy(), n


@pytest.mark.parametrize("pose", ["input", "orbit", "behind"])
@pytest.mark.parametrize("cam", ["vga", "odd", "negative_fy"])
def test_integrated_cloud_bit_exact(integrated, pose, cam):
    st, rec, rows, n = integrated
    T = {"input": st.frame_T_global[30], "orbit": orbit_pose(st, 30, 35.0, 0.4), "behind": BEHIND}[pose]
    cam = OUTPUT_CAMERAS[cam]
    out = rec.render(T, near=NEAR, far=FAR, **cam)
    torch.cuda.synchronize()
    ref = walk(rows, T, **cam)
    assert_bit_equal(out, ref)
    assert (ref["index"] != 0xFFFFFFFF).mean() > 0.2
    # the empty key raster is restored: a second render gives the same images
    again = rec.render(T, near=NEAR, far=FAR, **cam)
    assert_bit_equal(again, ref)


def test_each_output_alone(integrated):
    st, rec, rows, n = integrated
    T = st.frame_T_global[20]
    ref = walk(rows, T, **ODD)
    for k in R.RENDER_OUTPUTS:
        out = rec.render(T, near=NEAR, far=FAR, outputs=(k,), **ODD)
        assert set(out) == {k}
        assert_bit_equal(out, ref, (k,))


def raw_render(rec, T, cam, bufs, near=NEAR, far=FAR):
    """sm_render_surfels through the C ABI; bufs: name -> tensor [H, >= W (, 3)] (None = NULL) or (pointer, pitch)."""
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
    return rec.lib.fn["render_surfels"](rec._h, torch.cuda.current_stream().cuda_stream, C.byref(p),
                                        T.ctypes.data_as(C.c_void_p), *args)


def test_pitched_outputs_keep_their_padding(integrated):
    st, rec, rows, n = integrated
    T = st.frame_T_global[25]
    H, W = ODD["height"], ODD["width"]
    pad = 7
    bufs = {"depth": torch.full((H, W + pad), -3.5, dtype=torch.float32, device="cuda"),
            "color": torch.full((H, W + pad, 3), 0xAB, dtype=torch.uint8, device="cuda"),
            "normal": torch.full((H, W + pad, 3), 9.25, dtype=torch.float32, device="cuda"),
            "index": torch.full((H, W + pad), 0x5A5A5A5A, dtype=torch.int32, device="cuda")}
    before = {k: v.clone() for k, v in bufs.items()}
    assert raw_render(rec, T, ODD, bufs) == _lib.SM_OK
    torch.cuda.synchronize()
    ref = walk(rows, T, **ODD)
    assert_bit_equal({k: v[:, :W] for k, v in bufs.items()}, ref)
    for k in bufs:
        assert torch.equal(bufs[k][:, W:], before[k][:, W:]), k


def test_render_only_reads_the_state(integrated):
    st, rec, rows, n = integrated
    before, n0, m0 = rec.dump_state()
    before = before.copy()
    for T in (st.frame_T_global[30], BEHIND):
        rec.render(T, near=NEAR, far=FAR, **VGA)
    after, n1, m1 = rec.dump_state()
    assert (n0, m0) == (n1, m1)
    assert np.array_equal(before.view(np.uint32), after.view(np.uint32))


def test_invalid_arguments_are_rejected_without_a_launch(integrated, product):
    st, rec, rows, n = integrated
    H, W = 8, 10
    ok = {"depth": torch.zeros((H, W), dtype=torch.float32, device="cuda")}
    cam = dict(width=W, height=H, fx=10.0, fy=10.0, cx=5.0, cy=4.0)
    T = IDENTITY
    assert raw_render(rec, T, cam, ok) == _lib.SM_OK
    torch.cuda.synchronize()
    nan, inf = float("nan"), float("inf")
    bad_cams = [dict(cam, width=0), dict(cam, height=-1), dict(cam, fx=0.0), dict(cam, fy=nan), dict(cam, fx=inf),
                dict(cam, cx=nan), dict(cam, cy=inf)]
    launches = product.fn["kernel_launch_count"]()
    for c in bad_cams:
        assert raw_render(rec, T, c, ok) == _lib.SM_ERR_INVALID_ARGUMENT, c
    for near, far in [(0.0, 1.0), (-1.0, 1.0), (1.0, 1.0), (2.0, 1.0), (nan, 1.0), (0.1, nan)]:
        assert raw_render(rec, T, cam, ok, near, far) == _lib.SM_ERR_INVALID_ARGUMENT, (near, far)
    for k in range(12):
        Tb = IDENTITY.copy().reshape(-1)
        Tb[k] = nan if k % 2 else inf
        assert raw_render(rec, Tb, cam, ok) == _lib.SM_ERR_INVALID_ARGUMENT, k
    assert raw_render(rec, T, cam, {}) == _lib.SM_ERR_INVALID_ARGUMENT
    base = {"depth": 4 * W, "color": 3 * W, "normal": 12 * W, "index": 4 * W}
    big = torch.zeros(H * W * 16, dtype=torch.uint8, device="cuda")
    for k, row in base.items():
        assert raw_render(rec, T, cam, {k: (big.data_ptr(), row - 1)}) == _lib.SM_ERR_INVALID_ARGUMENT, k
        assert raw_render(rec, T, cam, {k: (big.data_ptr(), row)}) == _lib.SM_OK, k
        launches += 3
    torch.cuda.synchronize()
    assert product.fn["kernel_launch_count"]() == launches
    assert rec.lib.fn["render_surfels"](rec._h, None, None, T.ctypes.data_as(C.c_void_p), *([None, 0] * 4)) == \
        _lib.SM_ERR_INVALID_ARGUMENT


def test_render_between_session_pushes():
    st = S.make_stream(CAM, 40, device="cuda")
    pp, ip = params()
    rec = make()
    seen = []

    def between(f, status):
        if f not in (20, 33):
            return
        T = st.frame_T_global[int(status.last_integrated_frame)]
        out = rec.render(T, near=NEAR, far=FAR, **VGA)
        rows, n, merges = rec.dump_state()
        count = rec.surfel_count()
        other = make()
        other.load_state(rows, merges)
        again = other.render(T, near=NEAR, far=FAR, **VGA)
        torch.cuda.synchronize()
        assert_bit_equal(out, {k: v.cpu().numpy() for k, v in again.items()})
        idx = out["index"].cpu().numpy()
        distinct = np.unique(idx[idx >= 0])
        assert 0 < distinct.size <= count
        seen.append(f)
        other.close()

    with rec.session(pp, ip, (CAM.width, CAM.height)) as s:
        for f in range(st.frame_count):
            status = s.push(st.depth[f], st.color[f], st.global_T_frame[f], st.frame_T_global[f])
            between(f, status)
    assert seen == [20, 33]


# Rendered from the input pose of frame 40 after frames 4..43 of the 48-frame VGA stream, against the float64 ray
# cast of that pose. Measured on an H100 80GB HBM3 (700 W power limit):
#   nominal noise: median |d| 0.71 mm, p95 5.15 mm, coverage 0.520
#   noise free:    median |d| 0.62 mm, p95 5.15 mm, coverage 0.521
# The p95 hardly depends on the noise: it comes from disks at silhouettes and grazing surfaces, which reach past
# the surface they sample. Coverage is about half because the pre-processing drops depth beyond 3 m (max_depth),
# so the far walls have no surfels. Limits: twice the measured median, 1.5 times the p95, coverage 0.03 below.
SCENE_LIMITS = {
    None: dict(median=0.0015, p95=0.0078, coverage=0.49),
    0.0: dict(median=0.0013, p95=0.0078, coverage=0.49),
}


@pytest.mark.parametrize("sigma", [None, 0.0], ids=["nominal_noise", "noise_free"])
def test_rendered_depth_matches_the_scene(sigma):
    st = S.make_stream(CAM, 48, sigma_depth=sigma, device="cuda")
    pp, ip = params()
    rec = make()
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    f = last - 4
    pose64 = torch.from_numpy(S.trajectory(st.frame_count)[f]).to("cuda")
    gt, _ = S._raycast(CAM, pose64, "cuda")
    out = rec.render(st.frame_T_global[f], near=NEAR, far=FAR, outputs=("depth",), **VGA)
    depth = out["depth"].double()
    gt_valid = torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0)
    both = gt_valid & (depth > 0)
    err = (depth - gt)[both].abs().cpu().numpy()
    median, p95 = float(np.median(err)), float(np.percentile(err, 95))
    coverage = float(both.sum()) / float(gt_valid.sum())
    print(f"scene sigma={sigma}: median |d| {median:.6f} m, p95 {p95:.6f} m, coverage {coverage:.5f}")
    lim = SCENE_LIMITS[sigma]
    assert median <= lim["median"] and p95 <= lim["p95"] and coverage >= lim["coverage"]
