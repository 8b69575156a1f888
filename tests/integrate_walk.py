"""ctypes loader for tests/integrate_walk.c (TEST INFRASTRUCTURE) and the contract the host and GPU tests hold a frame to.

The product's association is reproducible, and sm_download_rasters hands out its decoded winners. GIVEN those
rasters (supporting surfel, count, conflicting surfel, first depth), everything else one Integrate() does is a plain
function of the state before the frame and the frame's inputs: merge flags, integrated / replaced / merged rows,
neighbour links, new-surfel flags, indices and rows, the counters. integrate_walk.c states that function
sequentially, one slot at a time, from the reference's kernels; it has none of the product's gather levels, lists
or short cuts. `walk()` runs it, `hold()` compares a run with it.

What is exact and what is bounded
---------------------------------
Every fmul / fadd / ffma of sm_math.cuh is an IEEE operation; the C file repeats them in the same order with
-ffp-contract=off and flushes denormal operands and results to zero as FTZ does. The SFU steps are not
reproducible: rcp in the projection, in the merge's radius ratio, in the integration weight and normalisation, in
the scale gate and in 1 / (count + 1) at creation; rsqrt of the integrated normal and of |p| in the facing test;
sqrt in the z of a measurement normal. The walk uses the correctly rounded value r for each and assumes the SFU
returns r (1 + d), |d| <= 2 ulp = 2^-22 (the documented errors are 1 ulp for rcp and sqrt, 2 ulp for rsqrt); the
reciprocal of a power of two is exact on both.

*Clear.* A discrete decision is `clear` when it is the same for every SFU result moved by -2 .. +2 ulp: the
projected pixel and its secondary pixel, the normal-compatibility test in the merge, the 1.44 / 0.694 ratio gates,
the 2.25 scale gate. A decision that compares values which already carry a bound (below) is clear when the two
sides are further apart than the bounds allow. A slot with an unclear merge or integration decision is not
compared at all, and its position bound is infinite, so whatever reads its position is unclear too; a slot with an
unclear link decision (or a link to an unclear slot) is compared except for its links.

*Bounds.* One integration computes p' = norm (g w + c p) with w = rcp(count), norm = rcp(w + c). With both
reciprocals off by 2^-22 and three roundings of 2^-24, |dp'| <= (2 * 2^-22 + 3 * 2^-24) (|g| w + c |p|) norm
<= 5.5 * 2^-23 max(|g|, |p|); the walk allows 8 * 2^-23 max(|g|_inf, |p|_inf) per integration and adds the bounds
of the two pixels (the second step's factor c norm is below 1). The same expression with a unit-length result
gives 16 * 2^-23 per integration for the normal (its rsqrt adds 2^-22, the square root in the measurement normal
2^-22); the confidence w + c carries 8 * 2^-23 (w + c). A colour channel is an integer: the walk evaluates it for
weight and normalisation each moved by -2, 0, +2 ulp (and for every value the first pixel's integration could have
left) and returns the range [lo, hi]; at an exact .5 the range is one value when weight and normalisation are
powers of two. The initial smooth position of a new surfel is (g + sum) rcp(k): 4 * 2^-23 |s|_inf, and 0 for k = 1.

*Bit for bit.* Everything that passes no SFU step: the position of a replaced or created surfel (and the smooth
position of a replacement), stamps, links, flag bytes, colours of created and replaced surfels, radii, a merged
slot's rows, every row of a slot the frame does not touch. The normal of a created or replaced surfel passes the
square root of the measurement normal: bound 4 * 2^-23.

The reference applies a merge in place while other threads still read the merged partner's radius, the product and
the walk decide every merge on the state before the frame. `status & ST_MERGE_CHAIN` marks the slots whose partner
merges in the same frame: the only ones where the reference may differ (it then does not merge them).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess
import tempfile
from pathlib import Path
from types import SimpleNamespace

import numpy as np

SOURCE = Path(__file__).resolve().parent / "integrate_walk.c"
ROW_COUNT = 25
INVALID = 0xFFFFFFFF
ST_UNCLEAR, ST_LINKS_UNCLEAR, ST_TOUCHED, ST_REPLACED, ST_INTEGRATED, ST_MERGE_UNCLEAR, ST_MERGE_CHAIN = 1, 2, 4, 8, 16, 32, 64
LINK_ROWS = slice(19, 23)


def _enum(name_prefix, text, name="Branch"):
    body = re.search(rf"enum {name} \{{(.*?)\}}", text, re.S).group(1)
    body = re.sub(r"//.*", "", body)
    return [t.strip() for t in body.split(",") if t.strip().startswith(name_prefix)]


_TEXT = SOURCE.read_text()
BRANCHES = [b[2:].lower() for b in _enum("B_", _TEXT) if b != "B_NUM"]
MUTATIONS = {m.group(1).lower(): 1 << int(m.group(2)) for m in re.finditer(r"\bMUT_(\w+) = 1 << (\d+)", _TEXT)}
# the front half (iw_associate, iw_blend): its own counters and mutations
FRONT_BRANCHES = [b[2:].lower() for b in _enum("F_", _TEXT, "FrontBranch") if b != "F_NUM"]
FRONT_MUTATIONS = {m.group(1).lower(): 1 << int(m.group(2)) for m in re.finditer(r"\bFM_(\w+) = 1 << (\d+)", _TEXT)}
ASSOCIATION_MUTATIONS = ("px_gt0", "min_depth_primary_only", "inactive_associate", "occlusion_ge", "radius_ge0",
                         "normal_test_always", "no_merge_conflict")
BLEND_MUTATIONS = tuple(m for m in FRONT_MUTATIONS if m not in ASSOCIATION_MUTATIONS)
SECONDARY_BIT = 0x80000000


class Params(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float),
                ("cy", C.c_float), ("depth_scaling", C.c_float), ("sensor_noise_factor", C.c_float),
                ("max_surfel_confidence", C.c_float), ("radius_factor", C.c_float), ("normal_threshold_deg", C.c_float),
                ("active_window", C.c_int32), ("frame_index", C.c_uint32), ("global_T_local", C.c_float * 12),
                ("local_T_global", C.c_float * 12), ("mutations", C.c_uint32)]


_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(SOURCE.read_bytes()).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"integrate_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"libintegrate_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the integration walk")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-o", str(tmp), str(SOURCE),
                            "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
        _lib.iw_integrate.restype = C.c_uint64
        _lib.iw_integrate.argtypes = [C.POINTER(Params), C.c_uint64, C.c_uint64] + [C.c_void_p] * 22
        _lib.iw_associate.restype = None
        _lib.iw_associate.argtypes = [C.POINTER(Params), C.c_uint64] + [C.c_void_p] * 17
        _lib.iw_blend.restype = None
        _lib.iw_blend.argtypes = [C.POINTER(Params), C.c_int] + [C.c_void_p] * 14
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def invert_rigid(m):
    m = np.asarray(m, np.float64).reshape(3, 4)
    r = m[:, :3].T
    return np.concatenate([r, (-r @ m[:, 3])[:, None]], 1).astype(np.float32)


def walk(rows_before, frame, rasters, camera, ip, frame_index, global_T_local, local_T_global=None, mutations=()):
    """One Integrate() after association. rows_before: [25, n] float32; frame: dict with depth_pre, depth (the blended
    depth the call left behind), normals [H, W, 2], radius, color [H, W, 3]; rasters: what download_rasters returns;
    camera: (W, H, fx, fy, cx, cy); ip: IntegrateParams. Returns the rows after the frame and per-slot status / bounds."""
    W, H, fx, fy, cx, cy = camera
    P = W * H
    rows_before = np.asarray(rows_before, np.float32)
    n = rows_before.shape[1]
    g = np.asarray(global_T_local, np.float32).reshape(-1)[:12]
    l = (invert_rigid(g) if local_T_global is None else np.asarray(local_T_global, np.float32)).reshape(-1)[:12]
    mut = 0
    for name in mutations:
        mut |= MUTATIONS[name]
    p = Params(W, H, fx, fy, cx, cy, ip.depth_scaling, ip.sensor_noise_factor, ip.max_surfel_confidence,
               ip.radius_factor_for_regularization_neighbors, ip.normal_compatibility_threshold_deg,
               ip.surfel_integration_active_window_size, int(frame_index), (C.c_float * 12)(*g), (C.c_float * 12)(*l), mut)
    stride = n + P
    rows = np.zeros((ROW_COUNT, stride), np.float32)
    rows[:, :n] = rows_before
    arr = lambda key, dtype, src=frame: np.ascontiguousarray(np.asarray(src[key]).reshape(-1), dtype)
    inputs = [arr("depth_pre", np.uint16), arr("depth", np.uint16), arr("normals", np.float32), arr("radius", np.float32),
              arr("color", np.uint8), arr("supporting_surfels", np.uint32, rasters),
              arr("supporting_surfel_counts", np.uint32, rasters), arr("conflicting_surfels", np.uint32, rasters),
              arr("first_surfel_depth", np.float32, rasters)]
    assert all(a.size == P * k for a, k in zip(inputs, (1, 1, 2, 1, 3, 1, 1, 1, 1)))
    out = SimpleNamespace(
        merge_flag=np.zeros(max(n, 1), np.uint8), new_flag=np.zeros(P, np.uint8), new_index=np.zeros(P, np.uint32),
        status=np.zeros(stride, np.uint8), pbound=np.zeros(stride, np.float32), nbound=np.zeros(stride, np.float32),
        cbound=np.zeros(stride, np.float32), color_lo=np.zeros(stride, np.uint32), color_hi=np.zeros(stride, np.uint32))
    branch = np.zeros(len(BRANCHES) + 1, np.uint64)
    counts = np.zeros(3, np.uint64)
    scratch = np.zeros((ROW_COUNT, max(n, 1)), np.float32)
    n_after = load().iw_integrate(C.byref(p), n, stride, _p(rows), *[_p(a) for a in inputs], _p(out.merge_flag),
                                  _p(out.new_flag), _p(out.new_index), _p(out.status), _p(out.pbound), _p(out.nbound),
                                  _p(out.cbound), _p(out.color_lo), _p(out.color_hi), _p(branch), _p(counts), _p(scratch))
    assert n_after <= stride
    for k in ("status", "pbound", "nbound", "cbound", "color_lo", "color_hi"):
        setattr(out, k, getattr(out, k)[:n_after])
    out.merge_flag = out.merge_flag[:n]
    out.rows, out.n_before, out.n_after = rows[:, :n_after], n, int(n_after)
    out.merges, out.unclear_merges = int(counts[1]), int(counts[2])
    out.new_flag, out.new_index = out.new_flag.reshape(H, W), out.new_index.reshape(H, W)
    out.branch = {name: int(v) for name, v in zip(BRANCHES, branch)}
    return out


def _channels(word):
    return np.stack([(word >> s) & 0xFF for s in (0, 8, 16)]).astype(np.int64)


def hold(res, rows_before, rows_after, new_flag=None, new_index=None, excused=None, smooth=True, links_may_drop=False,
         label=""):
    """Holds a run (rows_after [25, n_after], its new-surfel rasters) to the walk's result `res`. `excused`: bool mask
    of slots not to compare (slots that link to one are not compared for links). links_may_drop: the run also regularised,
    which drops links (kernels.cu:2184-2192) and never adds one, so a link may be invalid where the walk has one. Returns a dict of counts; raises
    AssertionError with the first differing slots."""
    n, n_after = res.n_before, res.n_after
    assert rows_after.shape[1] == n_after, f"{label}: surfels_size {rows_after.shape[1]}, the walk says {n_after}"
    if new_flag is not None:
        assert np.array_equal(np.asarray(new_flag).reshape(res.new_flag.shape), res.new_flag), f"{label}: new-surfel flags"
        assert np.array_equal(np.asarray(new_index).reshape(res.new_index.shape), res.new_index), f"{label}: new-surfel indices"
    want, got = res.rows, np.asarray(rows_after, np.float32)
    wu, gu = want.view(np.uint32), got.view(np.uint32)
    skip = (res.status & ST_UNCLEAR) != 0
    if excused is not None:
        skip = skip | excused
    links_w, links_g = wu[LINK_ROWS], gu[LINK_ROWS]
    reads_skipped = np.zeros(n_after, bool)
    for links in (links_w, links_g):
        for row in links:
            ok = row < n_after
            reads_skipped |= ok & skip[np.where(ok, row, 0)]
    skip_links = skip | ((res.status & ST_LINKS_UNCLEAR) != 0) | reads_skipped
    bad = {}

    def check(name, wrong):
        wrong = wrong & ~skip
        if wrong.any():
            bad[name] = np.flatnonzero(wrong)[:8].tolist()

    merged_w, merged_g = want[7, :n] < 0, got[7, :n] < 0
    check("merge flag", np.pad(merged_w != merged_g, (0, n_after - n)))
    used = 0.0
    for name, rows_, bound in (("position", (0, 1, 2), res.pbound), ("normal", (8, 9, 10), res.nbound),
                               ("confidence", (6,), res.cbound)):
        b = bound if name != "position" else np.where(np.arange(n_after) < n, bound, 0)   # new slots: pbound is of the smooth mean
        for r in rows_:
            with np.errstate(invalid="ignore"):
                diff = np.abs(want[r].astype(np.float64) - got[r])
            exact = wu[r] == gu[r]
            check(f"{name} row {r}", ~exact & ~(diff <= b))
            sel = ~skip & (b > 0) & np.isfinite(b) & np.isfinite(diff)
            if sel.any():
                used = max(used, float((diff[sel] / b[sel]).max()))
    for r, name in ((7, "radius squared"), (17, "creation stamp"), (18, "last update stamp")):
        check(name, wu[r] != gu[r])
    check("flag byte", (wu[24] >> 24) != (gu[24] >> 24))
    c, lo, hi = _channels(gu[24]), _channels(res.color_lo), _channels(res.color_hi)
    check("colour", np.any((c < lo) | (c > hi), axis=0))
    if smooth:
        old = np.arange(n_after) < n
        replaced = (res.status & ST_REPLACED) != 0
        for r in (3, 4, 5):
            check(f"smooth row {r} (old slot)", old & (wu[r] != gu[r]))
            with np.errstate(invalid="ignore"):
                diff = np.abs(want[r].astype(np.float64) - got[r])
            check(f"smooth row {r} (new slot)", ~old & (wu[r] != gu[r]) & ~(diff <= res.pbound))
            sel = ~old & ~skip & (res.pbound > 0)
            if sel.any():
                used = max(used, float((diff[sel] / res.pbound[sel]).max()))
        assert not (replaced & ~old).any()
    differs = (links_w != links_g) & ((links_g != INVALID) | (not links_may_drop))
    wrong_links = np.any(differs, axis=0) & ~skip_links
    dropped = int(((links_w != links_g) & ~skip_links).sum()) - int((differs & ~skip_links).sum())
    if wrong_links.any():
        bad["links"] = np.flatnonzero(wrong_links)[:8].tolist()
    stats = dict(slots=n_after, new=n_after - n, unclear=int(((res.status & ST_UNCLEAR) != 0).sum()),
                 links_unclear=int((skip_links & ~skip).sum()), excused=int(excused.sum()) if excused is not None else 0,
                 links_dropped=dropped, bit_exact_normals=int(np.all(wu[8:11] == gu[8:11], axis=0).sum()), bound_used=round(used, 3))
    if bad:
        detail = []
        for name, slots in bad.items():
            i = slots[0]
            detail.append(f"{name}: slots {slots}; slot {i}: status {int(res.status[i])} walk {want[:, i].tolist()} run {got[:, i].tolist()}"
                          f" before {np.asarray(rows_before)[:, i].tolist() if i < n else 'new'}")
        raise AssertionError(f"{label}: differs from the walk ({stats})\n" + "\n".join(detail))
    return stats


# ---- the front half: projection, association and measurement blending -------------------------------------------

def _front_params(camera, ip, frame_index, local_T_global, mutations):
    W, H, fx, fy, cx, cy = camera
    mut = 0
    for name in mutations:
        mut |= FRONT_MUTATIONS[name]
    l = np.asarray(local_T_global, np.float32).reshape(-1)[:12]
    zeros = (C.c_float * 12)()
    return Params(W, H, fx, fy, cx, cy, ip.depth_scaling, ip.sensor_noise_factor, 0.0, 0.0,
                  ip.normal_compatibility_threshold_deg, ip.surfel_integration_active_window_size, int(frame_index), zeros,
                  (C.c_float * 12)(*l), mut)


def associate(rows, depth_pre, normals, camera, ip, frame_index, local_T_global, mutations=()):
    """The association rasters one Integrate() builds from the state before the frame (rows [25, n]) and the pre-blend
    depth and normals: the min depth, the supporter count, the supporter set (events sup_pixel / sup_key, key = slot |
    SECONDARY_BIT for a secondary-pixel association), the depth sum (exact `sum` and the bound any summation order
    keeps to), the legal conflicting surfels (`conflict_legal`: pixel * 2^32 + slot, sorted; `conflict_any`: the
    pixels that have one) and the pixels whose outcome an SFU result within 2 ulp could change (`unclear`)."""
    W, H = camera[0], camera[1]
    P = W * H
    rows = np.ascontiguousarray(rows, np.float32)
    n = rows.shape[1]
    depth_pre = np.ascontiguousarray(np.asarray(depth_pre).reshape(-1), np.uint16)
    normals = np.ascontiguousarray(np.asarray(normals).reshape(-1), np.float32)
    assert depth_pre.size == P and normals.size == 2 * P
    p = _front_params(camera, ip, frame_index, local_T_global, mutations)
    r = SimpleNamespace(first=np.empty(P, np.float32), counts=np.empty(P, np.uint32), sum_float=np.empty(P, np.float32),
                        sum=np.empty(P, np.float64), sum_abs=np.empty(P, np.float64), unclear=np.empty(P, np.uint8))
    ties = np.empty(P, np.uint32)
    sup_pixel, sup_key = np.empty(2 * n + 1, np.uint32), np.empty(2 * n + 1, np.uint32)
    conf_pixel, conf_surfel, conf_stage = np.empty(3 * n + 1, np.uint32), np.empty(3 * n + 1, np.uint32), np.empty(3 * n + 1, np.uint8)
    counts = np.zeros(2, np.uint64)
    branch = np.zeros(len(FRONT_BRANCHES) + 1, np.uint64)
    load().iw_associate(C.byref(p), n, _p(rows), _p(depth_pre), _p(normals), _p(r.first), _p(r.counts), _p(r.sum_float),
                        _p(r.sum), _p(r.sum_abs), _p(r.unclear), _p(ties), _p(sup_pixel), _p(sup_key), _p(conf_pixel),
                        _p(conf_surfel), _p(conf_stage), _p(counts), _p(branch))
    ns, nc = int(counts[0]), int(counts[1])
    r.sup_pixel, r.sup_key = sup_pixel[:ns], sup_key[:ns]
    conf_pixel, conf_surfel, conf_stage = conf_pixel[:nc], conf_surfel[:nc], conf_stage[:nc]
    # the merge kernel runs after the association: where it writes, its writes are the final ones
    merge_writes = np.zeros(P, bool)
    merge_writes[conf_pixel[conf_stage == 1]] = True
    legal = (conf_stage == 1) | ~merge_writes[conf_pixel]
    r.conflict_legal = np.unique(conf_pixel[legal].astype(np.uint64) << np.uint64(32) | conf_surfel[legal])
    r.conflict_any = np.zeros(P, bool)
    r.conflict_any[conf_pixel] = True
    r.merge_writes = merge_writes
    # any order of float additions of k terms lies within (k - 1) 2^-24 sum |z| of the exact sum; one or two terms:
    # fl(a + b) in either order
    r.sum_bound = np.maximum(r.counts.astype(np.float64) - 1, 0) * 2.0 ** -24 * r.sum_abs
    few = r.counts <= 2
    r.sum[few], r.sum_bound[few] = r.sum_float[few], 0.0
    r.unclear = r.unclear.astype(bool)
    r.branch = {name: int(v) for name, v in zip(FRONT_BRANCHES, branch)}
    r.shape = (H, W)
    return r


def plain_winners(res):
    """The plain rule's supporting surfel per pixel: the least (secondary bit, slot) of the pixel's supporters."""
    best = np.full(res.first.size, INVALID, np.uint32)
    np.minimum.at(best, res.sup_pixel, res.sup_key)
    return np.where(best == INVALID, best, best & np.uint32(~SECONDARY_BIT & 0xFFFFFFFF))


def supporter_pairs(res):
    return np.unique(res.sup_pixel.astype(np.uint64) << np.uint64(32) | (res.sup_key & np.uint32(0x7FFFFFFF)))


def _member(sorted_pairs, pixels, values):
    keys = pixels.astype(np.uint64) << np.uint64(32) | np.asarray(values, np.uint64)
    at = np.minimum(np.searchsorted(sorted_pairs, keys), max(sorted_pairs.size - 1, 0))
    return (sorted_pairs.size > 0) & (sorted_pairs[at] == keys) if sorted_pairs.size else np.zeros(keys.shape, bool)


def hold_association(res, rasters, winner="member", label=""):
    """Holds association rasters (download_rasters, or the recorded reference) to the walk `res` on its clear pixels:
    min depth bit for bit, counts, conflicting surfel a legal one (INVALID where there is none), depth sums within the
    order bound. winner: "plain" (the plain rule, bit for bit), "member" (one of the pixel's supporters), or None.
    Returns a dict of counts; raises AssertionError with the first differing pixels."""
    P = res.first.size
    get = lambda k, dt: np.asarray(rasters[k]).reshape(-1).astype(dt, copy=False)
    first, counts = get("first_surfel_depth", np.float32), get("supporting_surfel_counts", np.uint32)
    conflicting, sums = get("conflicting_surfels", np.uint32), get("supporting_surfel_depth_sums", np.float32)
    clear = ~res.unclear
    pixels = np.arange(P, dtype=np.uint32)
    bad = {}

    def check(name, wrong):
        wrong = wrong & clear
        if wrong.any():
            bad[name] = np.flatnonzero(wrong)[:8].tolist()

    check("min depth", first.view(np.uint32) != res.first.view(np.uint32))
    check("count", counts != res.counts)
    ok_conflict = np.where(res.conflict_any & (conflicting != INVALID),
                           _member(res.conflict_legal, pixels, conflicting), ~res.conflict_any & (conflicting == INVALID))
    check("conflicting surfel", ~ok_conflict)
    with np.errstate(invalid="ignore"):
        check("depth sum", ~(np.abs(sums.astype(np.float64) - res.sum) <= res.sum_bound))
    if winner is not None:
        supporting = get("supporting_surfels", np.uint32)
        if winner == "plain":
            check("supporting surfel (plain rule)", supporting != plain_winners(res))
        else:
            supported = res.counts > 0
            member = _member(supporter_pairs(res), pixels, np.where(supporting == INVALID, 0, supporting))
            check("supporting surfel", ~np.where(supported, (supporting != INVALID) & member, supporting == INVALID))
    stats = dict(pixels=P, unclear=int(res.unclear.sum()), supported=int((res.counts > 0).sum()),
                 contested=int((res.counts > 1).sum()), conflicts=int(res.conflict_any.sum()),
                 merge_stage_conflicts=int(res.merge_writes.sum()))
    if bad:
        W = res.shape[1]
        detail = []
        for name, pix in bad.items():
            i = pix[0]
            detail.append(f"{name}: pixels {pix}; pixel {i} (x {i % W}, y {i // W}): walk first {res.first[i]} count "
                          f"{res.counts[i]} sum {res.sum[i]} +- {res.sum_bound[i]}; run first {first[i]} count {counts[i]} "
                          f"sum {sums[i]} conflicting {conflicting[i]}")
        raise AssertionError(f"{label}: association differs from the walk ({stats})\n" + "\n".join(detail))
    return stats


def blend(depth_pre, counts, sums, radius, depth_scaling, mutations=()):
    """The blended depth of BlendMeasurementsCUDA from the pre-blend depth [H, W] and the association's counts and
    depth sums as handed in. Returns depth, lo, hi ([H, W] u16: the depths the reciprocal bounds allow; lo == hi:
    exact), level_counts [2, radius + 1] (pixels per ring and level) and the branch counters."""
    depth_pre = np.ascontiguousarray(depth_pre, np.uint16)
    H, W = depth_pre.shape
    P = W * H
    counts = np.ascontiguousarray(np.asarray(counts).reshape(-1), np.uint32)
    sums = np.ascontiguousarray(np.asarray(sums).reshape(-1), np.float32)
    assert counts.size == P and sums.size == P and radius >= 1
    ip = SimpleNamespace(depth_scaling=depth_scaling, sensor_noise_factor=0.0, normal_compatibility_threshold_deg=0.0,
                         surfel_integration_active_window_size=0)
    p = _front_params((W, H, 1.0, 1.0, 0.0, 0.0), ip, 0, np.zeros(12), mutations)
    out, lo, hi = (np.empty(P, np.uint16) for _ in range(3))
    dist = [np.empty(P, np.uint8) for _ in range(2)]
    delta = [np.empty(P, np.float32) for _ in range(2)]
    bound = [np.empty(P, np.float64) for _ in range(2)]
    level_counts = np.zeros((2, radius + 1), np.uint64)
    branch = np.zeros(len(FRONT_BRANCHES) + 1, np.uint64)
    load().iw_blend(C.byref(p), int(radius), _p(depth_pre), _p(counts), _p(sums), _p(out), _p(lo), _p(hi), _p(dist[0]),
                    _p(dist[1]), _p(delta[0]), _p(delta[1]), _p(bound[0]), _p(bound[1]), _p(level_counts), _p(branch))
    return SimpleNamespace(depth=out.reshape(H, W), lo=lo.reshape(H, W), hi=hi.reshape(H, W),
                           level_counts=level_counts.astype(np.int64),
                           branch={name: int(v) for name, v in zip(FRONT_BRANCHES, branch)})


def hold_blend(res, depth, label=""):
    """Holds a blended depth [H, W] to the walk `res`: bit for bit where lo == hi, inside [lo, hi] elsewhere. Returns a
    dict of counts; raises AssertionError with the first differing pixels."""
    depth = np.asarray(depth).reshape(res.depth.shape).astype(np.int64)
    exact = res.lo == res.hi
    wrong = np.where(exact, depth != res.depth, (depth < res.lo) | (depth > res.hi))
    stats = dict(pixels=int(depth.size), blended=int((res.depth != 0).sum()), ranged=int((~exact).sum()),
                 levels=[int((row > 0).sum()) for row in res.level_counts])
    if wrong.any():
        ys, xs = np.nonzero(wrong)
        detail = [f"(x {x}, y {y}): run {depth[y, x]}, walk {res.depth[y, x]} [{res.lo[y, x]}, {res.hi[y, x]}]"
                  for y, x in list(zip(ys, xs))[:8]]
        raise AssertionError(f"{label}: blended depth differs from the walk at {int(wrong.sum())} pixels ({stats})\n"
                             + "\n".join(detail))
    return stats
