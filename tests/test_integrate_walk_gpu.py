"""One Integrate() on constructed states, held to the sequential restatement (tests/integrate_walk.c) fed with that
run's own association rasters: merge flags, rows, links, new-surfel rasters and counters without an envelope.

Both tie-breaks run every case: they pick different winners on contested pixels, and both must satisfy the same
function of their own winners."""
import numpy as np
import pytest
import torch

from surfelmeshing_b200 import reconstruction as R
from tests import integrate_walk as IW
from tests.test_integrate_walk_host import CASES, build_case, integrate_params
from tests.util import check_state_invariants, dev

pytestmark = pytest.mark.gpu

META_DETACH = 0x80000000


@pytest.mark.parametrize("plain_tiebreak", [False, True], ids=["wave", "plain"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_frame_is_the_walk_of_its_own_winners(product, case, plain_tiebreak):
    name, camera, frame_index, window, per_pixel, blending = case
    W, H, fx, fy, cx, cy = camera
    ip = integrate_params(window, blending)
    rows, frame, g32, l32 = build_case(camera, frame_index, window, per_pixel)
    n = rows.shape[1]
    rec = R.CUDASurfelReconstruction(n + W * H, W, H, fx, fy, cx, cy, lib=product)
    if plain_tiebreak:
        rec.configure("tiebreak_wave", 0)
    rec.load_state(rows, 3)
    loaded, _, _ = rec.dump_state()
    loaded = loaded.copy()
    depth = dev(frame["depth_pre"])
    rec.integrate(None, frame_index, ip, depth, dev(frame["normals"]), dev(frame["radius"]), dev(frame["color"]), g32, l32)
    torch.cuda.synchronize()
    after, n_after, merges = rec.dump_state()
    rasters = rec.download_rasters()
    blended = depth.cpu().numpy()
    assert blending or np.array_equal(blended, frame["depth_pre"])
    res = IW.walk(rows, dict(frame, depth=blended), rasters, camera, ip, frame_index, g32, l32)
    stats = IW.hold(res, rows, after, rasters["new_surfel_flag_vector"], rasters["new_surfel_indices"], label=name)
    print(f"{name} [{'plain' if plain_tiebreak else 'wave'}]: {stats}, merges {merges - 3} (walk {res.merges}, "
          f"unclear {res.unclear_merges})")
    assert rec.surfels_size() == res.n_after == n_after
    assert abs((merges - 3) - res.merges) <= res.unclear_merges
    assert stats["unclear"] <= 0.005 * n_after and stats["links_unclear"] <= 0.08 * n_after
    assert res.merges > 50 and stats["new"] > 50

    # rows the frame must not touch; the bookkeeping rows
    au, lu = after.view(np.uint32), loaded.view(np.uint32)
    clear = (res.status[:n] & IW.ST_UNCLEAR) == 0
    untouched = clear & ((res.status[:n] & IW.ST_TOUCHED) == 0) & (res.merge_flag == 0)
    for r in (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 17, 18, 24):
        assert np.array_equal(au[r, :n][untouched], lu[r, :n][untouched]), f"row {r} of a slot the frame does not touch"
    merged_now = clear & (res.merge_flag == 1)
    epochs = np.unique(au[14, :n][merged_now])
    assert len(epochs) == 1 and epochs[0] != 0, "row 14 of a slot merged by this frame holds the operation epoch"
    assert not au[14, :n][clear & (res.merge_flag == 0)].any()
    for r in (0, 1, 2, 3, 4, 5, 6, 8, 9, 10, 17):
        assert np.array_equal(au[r, :n][merged_now], lu[r, :n][merged_now]), f"row {r} of a merged slot"
    # the meta word of the regularisation records: the stamp, and the detach flag in bit 31
    all_clear = (res.status & IW.ST_UNCLEAR) == 0
    meta = (au[18] & ~np.uint32(META_DETACH)) | np.where((au[24] >> 24) == 1, np.uint32(META_DETACH), np.uint32(0))
    assert np.array_equal(au[15][all_clear], meta[all_clear])
    check_state_invariants(after, n_after)
    rec.close()
