"""The front half of one Integrate() - k_clear, k_project, k_associate, k_merge's conflicting-surfel write and k_blend -
held to its sequential restatement (tests/integrate_walk.c: iw_associate, iw_blend) on constructed states, and the
frame as a whole held from the state before it to the state after it (iw_associate / iw_blend here, iw_integrate
given the run's own rasters).

Grid: blend radii 1, 2, 3, 12, 17, 18, 33, 34, 39 (k_blend's x-halo grows at 17 -> 18 and 33 -> 34; 39 is the largest
radius its shared memory takes), frames smaller than one k_blend tile, one short of, exactly at and one past a tile,
odd, flipped, VGA and 1280 x 960; depth buffers pitched or not 16-byte aligned (k_blend's scalar path); surfel counts
on both sides of a multiple of 1024. Both tie-breaks: the plain rule is held bit for bit, the wave rule as one of the
supporters, identical over two runs."""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import reconstruction as R
from surfelmeshing_b200._lib import SM_ERR_INVALID_ARGUMENT, SurfelError
from tests import integrate_walk as IW
from tests.test_association_walk_host import CASES, TILE, front_case, front_params
from tests.util import dev

pytestmark = pytest.mark.gpu

PITCHED = {"tile-past-r18", "odd-r33", "flipped-r34"}   # the depth view starts 2 bytes into a wider row


def depth_buffer(depth, pitched):
    if not pitched:
        return dev(depth)
    H, W = depth.shape
    wide = dev(np.full((H, W + 24), 0xBEEF, np.uint16))
    view = wide[:, 1:1 + W]
    view.copy_(dev(depth))
    assert view.data_ptr() % 16 == 2
    return view


def run_frame(product, rows, frame, camera, ip, frame_index, g32, l32, plain, pitched):
    W, H, fx, fy, cx, cy = camera
    rec = R.CUDASurfelReconstruction(rows.shape[1] + W * H, W, H, fx, fy, cx, cy, lib=product)
    try:
        if plain:
            rec.configure("tiebreak_wave", 0)
        rec.load_state(rows, 3)
        depth = depth_buffer(frame["depth_pre"], pitched)
        rec.integrate(None, frame_index, ip, depth, dev(frame["normals"]), dev(frame["radius"]), dev(frame["color"]), g32, l32)
        torch.cuda.synchronize()
        return rec.download_rasters(), depth.cpu().numpy(), rec.dump_state()
    finally:
        rec.close()


@pytest.mark.parametrize("plain_tiebreak", [False, True], ids=["wave", "plain"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_front_half_is_the_walk(product, case, plain_tiebreak):
    name, camera, frame_index, window, per_pixel, radius, offset = case
    ip = front_params(window, radius)
    rows, frame, g32, l32 = front_case(camera, frame_index, window, per_pixel, offset)
    label = f"{name} [{'plain' if plain_tiebreak else 'wave'}]"
    rasters, blended, (after, n_after, _) = run_frame(product, rows, frame, camera, ip, frame_index, g32, l32,
                                                      plain_tiebreak, name in PITCHED)
    assoc = IW.associate(rows, frame["depth_pre"], frame["normals"], camera, ip, frame_index, l32)
    a_stats = IW.hold_association(assoc, rasters, winner="plain" if plain_tiebreak else "member", label=label)
    if not plain_tiebreak:   # the wave rule is reproducible too (the depth sums are float atomics: not compared)
        again, _, _ = run_frame(product, rows, frame, camera, ip, frame_index, g32, l32, False, name in PITCHED)
        for k in ("supporting_surfels", "supporting_surfel_counts", "first_surfel_depth"):
            assert np.array_equal(rasters[k], again[k]), f"{label}: {k} of a second run"
    # the blend, from this run's own counts and depth sums
    b = IW.blend(frame["depth_pre"], rasters["supporting_surfel_counts"], rasters["supporting_surfel_depth_sums"], radius,
                 ip.depth_scaling)
    b_stats = IW.hold_blend(b, blended, label=label)
    assert b.branch["start_depth_zero"] == 0
    # the rest of the frame, from the same rasters: the state before the frame held to the state after it
    res = IW.walk(rows, dict(frame, depth=blended), rasters, camera, ip, frame_index, g32, l32)
    i_stats = IW.hold(res, rows, after, rasters["new_surfel_flag_vector"], rasters["new_surfel_indices"], label=label)
    print(f"{label}: n {rows.shape[1]}, association {a_stats}, blend {b_stats}, frame {i_stats}")
    assert n_after == res.n_after
    assert a_stats["unclear"] <= 0.005 * a_stats["pixels"] and b_stats["ranged"] <= 0.005 * b_stats["pixels"]
    assert a_stats["supported"] > 0 and b_stats["levels"][0] + b_stats["levels"][1] > 0


def test_blend_radius_40_is_refused_before_any_launch(product):
    """39 is the largest radius whose tile region fits k_blend's shared memory; 40 is refused with
    SM_ERR_INVALID_ARGUMENT before any kernel of the frame runs (rasters, state and depth stay as they were), and the
    handle integrates afterwards."""
    camera = TILE
    W, H, fx, fy, cx, cy = camera
    window, frame_index = 2**31 - 1, 1000
    rows, frame, g32, l32 = front_case(camera, frame_index, window, 2.0)
    rec = R.CUDASurfelReconstruction(rows.shape[1] + 4 * W * H, W, H, fx, fy, cx, cy, lib=product)
    try:
        rec.load_state(rows, 3)
        inputs = (dev(frame["normals"]), dev(frame["radius"]), dev(frame["color"]), g32, l32)
        rec.integrate(None, frame_index, front_params(window, 39), dev(frame["depth_pre"]), *inputs)
        torch.cuda.synchronize()
        rasters, state = rec.download_rasters(), rec.dump_state()
        depth = dev(frame["depth_pre"])
        with pytest.raises(SurfelError) as refused:
            rec.integrate(None, frame_index + 1, front_params(window, 40), depth, *inputs)
        assert refused.value.code == SM_ERR_INVALID_ARGUMENT
        torch.cuda.synchronize()
        assert np.array_equal(depth.cpu().numpy(), frame["depth_pre"])
        after_refusal = rec.download_rasters()
        for k in rasters:
            assert np.array_equal(after_refusal[k], rasters[k]) or np.array_equal(after_refusal[k].view(np.uint32), rasters[k].view(np.uint32)), k
        rows_now, n_now, merges_now = rec.dump_state()
        assert n_now == state[1] and merges_now == state[2]
        assert np.array_equal(rows_now.view(np.uint32), state[0].view(np.uint32))
        # and the handle still integrates: the next frame is the walk of the state it starts from
        ip = front_params(window, 39)
        depth = dev(frame["depth_pre"])
        rec.integrate(None, frame_index + 1, ip, depth, *inputs)
        torch.cuda.synchronize()
        assoc = IW.associate(rows_now, frame["depth_pre"], frame["normals"], camera, ip, frame_index + 1, l32)
        rasters = rec.download_rasters()
        IW.hold_association(assoc, rasters, winner="member", label="after the refusal")
        b = IW.blend(frame["depth_pre"], rasters["supporting_surfel_counts"], rasters["supporting_surfel_depth_sums"], 39,
                     ip.depth_scaling)
        IW.hold_blend(b, depth.cpu().numpy(), label="after the refusal")
    finally:
        rec.close()
