"""One integrated frame of the frame loop held to the walks, given the state it started from (TEST INFRASTRUCTURE).

`hold_frame` chains what the suite already states about one Integrate() and adds no restatement of its own:

  association   IW.associate on the state before the frame and the frame's pre-blend depth and normals, held by
                IW.hold_association (winners bit for bit under the plain tie-break, one of the pixel's supporters
                under the wave tie-break);
  blending      IW.blend on the run's own counts and depth sums;
  the cycle     IW.walk fed with the run's association rasters and the walk's blended depth, held by IW.hold;
  regularising  with regularisation on, the smooth positions after the step are held to reg_walk.regularize chained
                over the step's sweeps (test_regularize_float64_gpu.expected_integrate / check), starting from the
                walk's post-cycle smooth positions and links and the run's other rows;
  counters      surfels_size, the merge count and sm_frame_counters' N, M and S.

The blended depth the run used is never observable
--------------------------------------------------
IW.blend gives each pixel a depth and the range [lo, hi] its reciprocal bounds allow; the walk is fed the depth. Where
lo == hi the run's depth is that value, so the walk is fed exactly what the run read. Where lo != hi (a ranged pixel)
the run read some value in [lo, hi]. Every slot that projects onto a ranged pixel reads it, winner of the pixel or
not: its integrate / occluded / conflicting decisions compare with it, and an integration or a replacement takes its
position from it. The walk is run twice more, with lo and with hi at every ranged pixel, and a slot is excused
(IW.hold(excused=)) where

  - its rows differ between those walks and the one fed the blended depth, or one of them finds it unclear: each
    decision is a comparison with the measurement that is monotone in it, so a slot whose decisions agree at both
    ends agrees everywhere between, and a slot whose position is taken from the depth differs between lo and hi;
  - it is a surfel created beside the pixel of a slot excused so: its link to that slot and the smooth mean it takes
    from it follow a distance test against the slot's integrated position, which is not monotone in the depth;
  - IW.hold itself leaves out the links of every slot that links to an excused one in either state, which covers a
    neighbour update or a new surfel's link decision that reads an excused slot's position or a ranged depth.

The new-surfel flag of a pixel is `depth > 0` on an interior pixel without supporter and conflicting surfel, so
whatever value in [lo, hi] the run read, its flags are those of the walk fed with lo or of the walk fed with hi. If
those two give different flags, the run's creation scan could differ from the walk's at one pixel and with it the
index of every later new surfel: the frame is excused as a whole and not compared. An excused frame does not break a
chain, which continues from the run's own state.

Chains
------
`Chain` holds frame after frame of one handle, each from the state the previous hold (or a call between pushes) left.
Its `Inputs` pre-process each pushed frame on a second handle, after a `stage` hook that restates on the CPU what the
frame loop's ring does to a raw frame before the pre-processing reads it: nothing (`stage_identity`), the input
pyramid of --pyramid_level (`stage_pyramid`) or the MedianFilterAndDensifyDepthMap passes (`stage_median`). The hook
is applied to the frame and to each of its outlier-filter neighbours. Frames and poses are indexed by push: a
pose-free session that leaves lost frames out pushes source frames `pushed_sources(states)`.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from tests import integrate_walk as IW
from tests.test_regularize_float64_gpu import check as check_sweeps, expected_integrate
from tests.util import other_frames

INVALID = IW.INVALID


def frame_counters(rec):
    """sm_frame_counters: (N slots swept, V visible, S sum of supporting counts, M new surfels)."""
    out = (C.c_uint64 * 4)()
    rec.lib.call("frame_counters", rec._h, None, C.byref(out))
    return tuple(int(v) for v in out)


def created_beside(res, rasters, excused):
    """New surfels whose creation reads the position of an `excused` slot: the supporter of one of their pixel's
    four neighbours."""
    H, W = res.new_flag.shape
    sup = np.asarray(rasters["supporting_surfels"]).reshape(H, W).astype(np.int64)
    valid = (sup != INVALID) & (sup < res.n_after)
    padded = np.zeros((H + 2, W + 2), bool)
    padded[1:-1, 1:-1] = valid & excused[np.where(valid, sup, 0)]
    near = padded[:-2, 1:-1] | padded[2:, 1:-1] | padded[1:-1, :-2] | padded[1:-1, 2:]
    out = np.zeros(res.n_after, bool)
    new = res.new_flag.astype(bool) & near
    out[res.n_before + res.new_index[new].astype(np.int64)] = True
    return out


def hold_frame(rows_before, rows_after, merge_count, rasters, frame, frame_index, global_T_local, local_T_global,
               camera, ip, merges_before=0, counters=None, winner="member", merge_chains_excused=False, label=""):
    """Holds one integrated frame. rows_before / rows_after: the dumped states [25, n] before and after it;
    merge_count: the merge count reported after it (merges_before: the one reported before it); rasters:
    download_rasters after it; frame: dict of the frame's pre-processed depth_pre [H, W] u16, normals [H, W, 2],
    radius [H, W] and color [H, W, 3]; counters: frame_counters() after it, or None; winner: "plain" under the plain
    tie-break, "member" otherwise; merge_chains_excused: the states come from the reference, which applies a merge in
    place (IW's ST_MERGE_CHAIN slots). Returns per-frame statistics; raises AssertionError at the first difference."""
    W, H = camera[0], camera[1]
    P = W * H
    rows_before = np.asarray(rows_before, np.float32)
    rows_after = np.asarray(rows_after, np.float32)
    n = rows_before.shape[1]
    get = lambda k: np.asarray(rasters[k]).reshape(H, W)
    counts = get("supporting_surfel_counts")

    # 1. association
    front = IW.associate(rows_before, frame["depth_pre"], frame["normals"], camera, ip, frame_index, local_T_global)
    IW.hold_association(front, rasters, winner=winner, label=f"{label} association")

    # 2. blending
    depth_pre = np.asarray(frame["depth_pre"]).reshape(H, W)
    if ip.do_blending:
        bl = IW.blend(depth_pre, counts, get("supporting_surfel_depth_sums"), ip.measurement_blending_radius,
                      ip.depth_scaling)
        depth, lo, hi = bl.depth, bl.lo, bl.hi
    else:
        depth = lo = hi = depth_pre
    ranged = lo != hi
    walk_frame = dict(frame, depth=depth)
    walk = lambda d: IW.walk(rows_before, dict(walk_frame, depth=d), rasters, camera, ip, frame_index,
                             global_T_local, local_T_global)
    res = walk(depth)
    stats = dict(pixels=P, unclear=int(front.unclear.sum()), ranged=int(ranged.sum()), slots=res.n_after,
                 excused=0, excused_frame=0, branch=res.branch, bound_used=0.0, merges=res.merges,
                 new=res.n_after - n)
    excused = np.zeros(res.n_after, bool)
    if ranged.any():
        ends = walk(np.where(ranged, lo, depth)), walk(np.where(ranged, hi, depth))
        if not np.array_equal(ends[0].new_flag, ends[1].new_flag):
            stats.update(excused_frame=1, branch={}, merges=0, new=0)
            return stats
        for end in ends:
            excused |= np.any(end.rows.view(np.uint32) != res.rows.view(np.uint32), axis=0)
            excused |= (end.status & IW.ST_UNCLEAR) != 0
        excused |= created_beside(res, rasters, excused)
    if merge_chains_excused:
        excused |= (res.status & IW.ST_MERGE_CHAIN) != 0
    stats["excused"] = int(excused.sum())

    # 3. the cycle, and the regularisation sweeps of the step
    regularising = ip.regularization_iterations_per_integration_iteration > 0
    held = IW.hold(res, rows_before, rows_after, rasters["new_surfel_flag_vector"], rasters["new_surfel_indices"],
                   excused=excused, smooth=not regularising, links_may_drop=regularising, label=label)
    stats["bound_used"] = held["bound_used"]
    if regularising:
        # the walk does not know the smooth position of an unclear or excused slot, nor the links of a slot with an
        # unclear link decision: check() leaves them out with the slots that read them
        unknown = excused | ((res.status & (IW.ST_UNCLEAR | IW.ST_LINKS_UNCLEAR)) != 0)
        start = rows_after.copy()
        start[3:6] = res.rows[3:6]
        start[IW.LINK_ROWS] = res.rows[IW.LINK_ROWS]
        new = np.arange(res.n_after) >= n
        error = np.where(new & ~unknown, np.sqrt(3) * res.pbound.astype(np.float64), 0.0)
        sweeps = expected_integrate(start, frame_index, ip, remove_below=n, input_error=error)
        reg = check_sweeps(start, rows_after, sweeps, f"{label} regularisation", excused=unknown)
        stats["bound_used"] = max(stats["bound_used"], reg["worst"])
        stats["reg_close"] = reg["close"]

    # 4. counters
    assert rows_after.shape[1] == res.n_after, f"{label}: surfels_size {rows_after.shape[1]}, the walk says {res.n_after}"
    allowance = res.unclear_merges + (int(((res.status[:n] & IW.ST_MERGE_CHAIN) != 0).sum()) if merge_chains_excused else 0)
    assert abs((int(merge_count) - int(merges_before)) - res.merges) <= allowance, \
        f"{label}: merge count {merge_count} after {merges_before}, the walk merges {res.merges} (unclear {res.unclear_merges})"
    if counters is not None:
        swept, _, support, created = counters
        assert swept == n and created == res.n_after - n, f"{label}: frame counters N {swept}, M {created}"
        assert support == int(counts.astype(np.int64).sum()), f"{label}: frame counters S {support}"
    return stats


class Totals:
    """Per-chain sums of hold_frame's statistics and the coverage floors every chain must reach."""
    FLOOR_BRANCHES = {"merges": ("merged",), "replacements": ("replace", "replace_then_second"),
                      "integrations": ("integrate_once", "integrate_twice"),
                      "conflicting surfels": ("conf_decrement", "replace", "replace_then_second")}

    def __init__(self, label):
        self.label = label
        self.frames = self.excused_frames = self.pixels = self.unclear = self.ranged = self.slots = self.excused = 0
        self.new = 0
        self.bound = 0.0
        self.branch = {}

    def add(self, s):
        self.frames += 1
        self.excused_frames += s["excused_frame"]
        self.pixels += s["pixels"]
        self.unclear += s["unclear"]
        self.ranged += s["ranged"]
        if s["excused_frame"]:
            return
        self.slots += s["slots"]
        self.excused += s["excused"]
        self.new += s["new"]
        self.bound = max(self.bound, s["bound_used"])
        for k, v in s["branch"].items():
            self.branch[k] = self.branch.get(k, 0) + v

    def floors(self):
        return {name: sum(self.branch.get(b, 0) for b in keys) for name, keys in self.FLOOR_BRANCHES.items()}

    def report(self):
        pct = lambda a, b: 100.0 * a / max(b, 1)
        return (f"{self.label}: {self.frames} frames held, {self.excused_frames} excused; unclear association "
                f"{pct(self.unclear, self.pixels):.3f} %, ranged blend {pct(self.ranged, self.pixels):.3f} %, excused "
                f"slots {pct(self.excused, self.slots):.3f} %; branches {dict(self.floors(), new=self.new)}; largest "
                f"bound used {self.bound:.3f}")

    def assert_fractions(self):
        assert self.unclear <= 0.005 * self.pixels, self.report()
        assert self.ranged <= 0.005 * self.pixels, self.report()
        assert self.excused <= 0.005 * self.slots, self.report()
        assert self.excused_frames * 10 <= max(self.frames, 10), self.report()

    def assert_floors(self, min_frames, waive=()):
        """waive: floors (FLOOR_BRANCHES names) a chain cannot reach at its size; the caller says why."""
        floors = self.floors()
        assert self.frames >= min_frames, f"{self.label}: {self.frames} frames held"
        assert all(v > 0 for k, v in floors.items() if k not in waive) and self.new > 0, \
            f"{self.label}: branches not reached {floors}"
        self.assert_fractions()


# ---------------------------------------------------------------------------------------------
# chains: the inputs of each pushed frame, and frame after frame of one handle
# ---------------------------------------------------------------------------------------------

def camera_tuple(cam):
    return cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy


def stage_identity(depth, color):
    """Frames read at the handle's size, as pushed."""
    return depth, color


def stage_pyramid(level, width, height):
    """--pyramid_level L (APP/main.cc:951-952, 973-981): the depth map downscaled by the median of each block without
    zeros straight to the handle's width x height, the colour image by L rounds of halving."""
    from tests import pyramid_walk as PW

    def stage(depth, color):
        return PW.downscale_median_excluding(depth, width, height), PW.color_image_pyramid(color, level)
    return stage


def stage_median(passes):
    """--median_filter_and_densify_iterations n (APP/main.cc:927-939): n passes over the depth map; colour as is."""
    from oracle import cpu_walk

    def stage(depth, color):
        for _ in range(passes):
            depth = cpu_walk.median_filter_and_densify(depth)
        return depth, color
    return stage


def pushed_sources(states, held_out=True):
    """The source frame of each push of a pose-free session from its per-frame states (TrackedSession.states): with
    relocalisation on (held_out), a frame left "lost" is not pushed, so push index and source frame diverge."""
    return [f for f, s in enumerate(states) if not (held_out and s == "lost")]


class Inputs:
    """The pre-processed inputs of the frames pushed into a handle, from a handle of their own (created on first use).

    depth / color: raw frames by source index (tensors or arrays, any device); sources: the source frame of each push
    (a list the caller may extend while the session runs; None: push p is source frame p); stage(raw_depth, raw_color)
    -> (depth, color) at `cam`, the handle's camera."""

    def __init__(self, cam, depth, color, pp, stage=stage_identity, sources=None):
        self.cam, self.depth, self.color, self.pp, self.stage = cam, depth, color, pp, stage
        self.sources = sources
        self.rec = None
        self.staged = {}

    def source(self, push):
        return push if self.sources is None else self.sources[push]

    def others(self, push):
        """The source frames of push `push`'s outlier-filter neighbours: the K/2 pushes before it and after it."""
        return [self.source(p) for p in other_frames(push, self.pp.outlier_filtering_frame_count)]

    def staged_frame(self, source):
        """Source frame `source` after the stage hook: (depth [H, W] uint16, colour [H, W, 3] uint8) numpy arrays."""
        if source not in self.staged:
            host = lambda a: a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
            self.staged[source] = self.stage(host(self.depth[source]), host(self.color[source]))
        return self.staged[source]

    def frame(self, push, global_T_frame, frame_T_global):
        """hold_frame's `frame` for push `push`; global_T_frame / frame_T_global: the poses pushed, by push index."""
        import torch
        from surfelmeshing_b200 import reconstruction as R
        cam, pp = self.cam, self.pp
        if self.rec is None:
            self.rec = R.CUDASurfelReconstruction(1024, *camera_tuple(cam))
        K = pp.outlier_filtering_frame_count
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        raw_depth, color = self.staged_frame(self.source(push))
        others = [dev(self.staged_frame(s)[0]) for s in self.others(push)]
        g = np.asarray(global_T_frame[:push + K // 2 + 1], np.float32)
        l = np.asarray(frame_T_global[:push + K // 2 + 1], np.float32)
        transforms = R.outlier_filter_transforms(g, l, push, K, pp.depth_scaling)
        H, W = cam.height, cam.width
        assert raw_depth.shape == (H, W) and color.shape == (H, W, 3), (raw_depth.shape, color.shape)
        d = torch.zeros((H, W), dtype=torch.uint16, device="cuda")
        n = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
        r = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        self.rec.preprocess(None, pp, dev(raw_depth), others, transforms, d, n, r)
        torch.cuda.synchronize()
        return dict(depth_pre=d.cpu().numpy(), normals=n.cpu().numpy(), radius=r.cpu().numpy(), color=color)

    def close(self):
        if self.rec is not None:
            self.rec.close()


class Chain:
    """Holds frame after frame of one handle, each from the state the previous hold (or a call between) left.
    poses: (global_T_frame, frame_T_global), the poses pushed, by push index (lists the caller may extend)."""

    def __init__(self, label, rec, inputs, ip, poses, first_frame_index=0, plain=False):
        self.label, self.rec, self.inputs, self.ip, self.poses = label, rec, inputs, ip, poses
        self.first = first_frame_index
        self.winner = "plain" if plain else "member"
        self.rows, self.merges = np.zeros((25, 0), np.float32), 0
        self.totals = Totals(label)

    def restart(self):
        """The state after a call between pushes, or after a frame not held: the next frame starts from it."""
        rows, _, merges = self.rec.dump_state()
        self.rows, self.merges = rows.copy(), merges

    def hold(self, frame_index):
        rec = self.rec
        push = frame_index - self.first
        rows, n, merges = rec.dump_state()
        rows = rows.copy()
        rasters = rec.download_rasters()
        counters = frame_counters(rec)
        g, l = self.poses
        stats = hold_frame(self.rows, rows, merges, rasters, self.inputs.frame(push, g, l), frame_index, g[push], l[push],
                           camera_tuple(self.inputs.cam), self.ip, merges_before=self.merges, counters=counters,
                           winner=self.winner, label=f"{self.label} frame {frame_index}")
        self.totals.add(stats)
        self.rows, self.merges = rows, merges

    def finish(self, min_frames, waive=()):
        self.inputs.close()
        print(self.totals.report())
        self.totals.assert_floors(min_frames, waive)
