#!/usr/bin/env python
"""The keyframe database and sm_relocalise on the VGA synthetic desk stream (bench.py's stream: stream_id 0, nominal
noise). Prints one JSON summary with the card's name and power limit (and writes it to --out).

1. Map: the first 150 frames integrated with their true poses (sm_stream_run).
2. Timing (host clock around the synchronous calls, median of --timed calls after warm-up): sm_keyframe_db_encode
   (CUDA events over a batch), sm_keyframe_db_add of a frame that is not stored (the per-frame cost of offering a
   frame) and sm_keyframe_db_query, each at 1 k and 4 k stored keyframes; sm_relocalise per attempt.
3. Keyframes per 100 frames: every frame of the --frames bench stream offered at its true pose, per add_fraction.
4. Kidnapped frames: --revisits frames at poses 1-3 cm and 0.5-2 degrees off mapped orbit poses, and --unmapped
   frames from the far side of the orbit, all with fresh noise. The database holds the mapped frames offered at
   their true poses. Every candidate of a query is tracked (as sm_relocalise would, in order) and recorded, so that
   the acceptance rule can be evaluated for any thresholds.

--sweep evaluates a grid of add_fraction x max_query_fraction x tracking parameters x candidates x acceptance
thresholds: the recovery rate and the worst error of the revisit frames (within 1 cm and 0.5 degrees counts as
recovered), and the false accepts (an accepted pose outside those bounds, revisit or unmapped). The defaults of
sm_default_reloc_params are the grid point with no false accept and the highest recovery, then the fewest
keyframes and candidates (track variants: sm_default_track_params with its 5 cm gate, a 10 cm gate, four levels).
Where grid points tie on all of these (max_query_fraction, accept_rms on the desk stream) the middle value is kept."""
import argparse
import ctypes as C
import itertools
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import _lib  # noqa: E402
from surfelmeshing_b200 import synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, RelocParams, TrackParams  # noqa: E402
from tests import reloc_walk as W  # noqa: E402

VGA = S.Camera.tum(640, 480)
MAX_T, MAX_R = 0.01, 0.5   # the pose-free bounds of tests/test_track_gpu.py::test_pose_free_stream


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"


def pose_error(a, b):
    a, b = np.asarray(a, np.float64).reshape(3, 4), np.asarray(b, np.float64).reshape(3, 4)
    Rr = a[:, :3] @ b[:, :3].T
    s = 0.5 * np.linalg.norm([Rr[2, 1] - Rr[1, 2], Rr[0, 2] - Rr[2, 0], Rr[1, 0] - Rr[0, 1]])
    return float(np.linalg.norm(a[:, 3] - b[:, 3])), math.degrees(math.atan2(s, (np.trace(Rr) - 1) / 2))


def timed(fn, n):
    out = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out))


def track_variants():
    base = TrackParams.defaults()
    wide = TrackParams.from_buffer_copy(base)
    wide.max_point_distance = 0.1
    deep = TrackParams.from_buffer_copy(base)
    deep.levels = 4
    deep.iterations = (C.c_int32 * 4)(4, 5, 10, 10)
    return {"gate_5cm": base, "gate_10cm": wide, "levels_4": deep}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--timed", type=int, default=50)
    ap.add_argument("--revisits", type=int, default=24)
    ap.add_argument("--unmapped", type=int, default=12)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--out", default="probe_out/reloc_probe.json")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    summary = {"card": card(), "defaults": {}}
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = VGA.valid_region_radius()
    ip = IntegrateParams.defaults()
    st = S.make_stream(VGA, args.frames, device="cuda")
    mapped = 150
    rec = R.CUDASurfelReconstruction(5_000_000, VGA.width, VGA.height, VGA.fx, VGA.fy, VGA.cx, VGA.cy)
    rec.stream_run(None, st.depth[:mapped].contiguous(), st.color[:mapped].contiguous(), st.global_T_frame[:mapped],
                   st.frame_T_global[:mapped], st.others_TR_reference[:mapped], pp, ip, 4, mapped - 4)
    torch.cuda.synchronize()
    defaults = RelocParams.defaults()
    summary["defaults"] = {k: (getattr(defaults, k) if k != "track" else "sm_default_track_params, max_point_distance 0.1")
                           for k, _ in defaults._fields_}

    # 2. timing
    big = RelocParams.from_buffer_copy(defaults)
    big.capacity = 4096
    db = R.KeyframeDatabase(rec, big)
    d0, c0 = st.depth[10], st.color[10]
    for _ in range(20):
        db.encode(d0, c0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        db.encode(d0, c0)
    e1.record()
    torch.cuda.synchronize()
    summary["encode_ms"] = e0.elapsed_time(e1) / 200
    timing = {}
    f = 0
    for target in (1000, 4096):
        while len(db) < target:   # distinct frames, forced: the stored codes are those of a real stream
            db.add(st.depth[f % args.frames], st.color[f % args.frames], st.global_T_frame[f % args.frames],
                   force=True)
            f += 1
        probe_d, probe_c = st.depth[7], st.color[7]   # stored already: add does not append
        timing[f"add_ms_{target}"] = timed(lambda: db.add(probe_d, probe_c, st.global_T_frame[7]), args.timed)
        timing[f"query_ms_{target}"] = timed(lambda: db.query(probe_d, probe_c), args.timed)
    db.close()
    small = R.KeyframeDatabase(rec, defaults)
    for k in range(4, mapped - 4):
        small.add(st.depth[k], st.color[k], st.global_T_frame[k])
    timing["keyframes_of_the_mapped_frames"] = len(small)
    timing[f"add_ms_{len(small)}"] = timed(lambda: small.add(st.depth[70], st.color[70], st.global_T_frame[70]),
                                           args.timed)
    summary["timing"] = timing

    # 3. keyframes per 100 frames
    per100 = {}
    for fraction in (0.05, 0.1, 0.15, 0.2, 0.3):
        p = RelocParams.from_buffer_copy(defaults)
        p.add_fraction = fraction
        d = R.KeyframeDatabase(rec, p)
        for k in range(args.frames):
            d.add(st.depth[k], st.color[k], st.global_T_frame[k])
        per100[str(fraction)] = 100.0 * len(d) / args.frames
        d.close()
    summary["keyframes_per_100_frames"] = per100

    # 4. kidnapped frames
    revisit_at = np.linspace(8, mapped - 8, args.revisits).astype(int).tolist()
    revisits = W.revisit_frames(VGA, revisit_at)
    far = np.linspace(400, 600, args.unmapped).astype(int).tolist()
    far_poses = S.trajectory(max(far) + 1)
    unmapped = [(*W.render_frame(VGA, far_poses[k], 900 + k), far_poses[k].astype(np.float32)) for k in far]

    def records(add_fraction, max_query_fraction, tp):
        """Per query frame: [(distance, tracked, inlier fraction, rms, t error, r error)] of every candidate."""
        p = RelocParams.from_buffer_copy(defaults)
        p.add_fraction, p.max_query_fraction, p.candidates = add_fraction, max_query_fraction, 8
        d = R.KeyframeDatabase(rec, p)
        for k in range(4, mapped - 4):
            d.add(st.depth[k], st.color[k], st.global_T_frame[k])
        tcl = TrackParams.from_buffer_copy(tp)
        out = []
        for depth, color, truth in revisits + unmapped:
            idx, dist = d.query(depth, color)
            rows = []
            for i, dd in zip(idx, dist):
                pose, res = rec.track(depth, d.pose(int(i)), params=tcl, pp=pp)
                et, er = pose_error(pose, truth)
                rows.append((int(dd), int(res.tracked), res.inliers / max(res.valid_pixels, 1), res.rms_residual,
                             et, er))
            out.append(rows)
        n = len(d)
        d.close()
        return n, out

    def evaluate(rows_per_frame, candidates, accept_fraction, accept_rms):
        recovered, false, worst, attempts = 0, 0, (0.0, 0.0), []
        for q, rows in enumerate(rows_per_frame):
            accepted = None
            tried = 0
            for dist, tracked, frac, rms, et, er in rows[:candidates]:
                tried += 1
                if tracked and frac >= accept_fraction and rms <= accept_rms:
                    accepted = (et, er)
                    break
            attempts.append(tried)
            if accepted is None:
                continue
            good = accepted[0] <= MAX_T and accepted[1] <= MAX_R
            if not good:
                false += 1
            elif q < len(revisits):
                recovered += 1
                worst = (max(worst[0], accepted[0]), max(worst[1], accepted[1]))
        return {"recovered": recovered / len(revisits), "false_accepts": false,
                "worst_mm": worst[0] * 1e3, "worst_deg": worst[1], "mean_attempts": float(np.mean(attempts))}

    # time per attempt with the defaults
    dflt = R.KeyframeDatabase(rec, defaults)
    for k in range(4, mapped - 4):
        dflt.add(st.depth[k], st.color[k], st.global_T_frame[k])
    per_attempt, outcomes = [], []
    for depth, color, truth in revisits + unmapped:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pose, res = rec.relocalise(dflt, depth, color, pp=pp)
        ms = (time.perf_counter() - t0) * 1e3
        if res.attempts:
            per_attempt.append((ms - timing[f"add_ms_{len(small)}"]) / res.attempts)
        outcomes.append((int(res.relocalised), *(pose_error(pose, truth) if res.relocalised else (None, None))))
    rev = outcomes[:len(revisits)]
    ok = [o for o in rev if o[0] and o[1] <= MAX_T and o[2] <= MAX_R]
    summary["relocalise_defaults"] = {
        "ms_per_attempt": float(np.median(per_attempt)) if per_attempt else None,
        "revisit_recovered": len(ok) / len(revisits),
        "revisit_worst_mm": max((o[1] for o in ok), default=0.0) * 1e3,
        "revisit_worst_deg": max((o[2] for o in ok), default=0.0),
        "revisit_median_mm": float(np.median([o[1] for o in ok])) * 1e3 if ok else None,
        "unmapped_accepted": sum(o[0] for o in outcomes[len(revisits):]),
        "false_accepts": sum(1 for o in outcomes if o[0] and not (o[1] <= MAX_T and o[2] <= MAX_R)),
    }
    dflt.close()

    if args.sweep:
        sweep = []
        for (add_fraction, max_query_fraction), (tname, tp) in itertools.product(
                [(0.05, 0.3), (0.1, 0.3), (0.1, 0.4), (0.2, 0.4), (0.2, 0.5), (0.3, 0.5)], track_variants().items()):
            keyframes, rows = records(add_fraction, max_query_fraction, tp)
            for candidates, accept_fraction, accept_rms in itertools.product((1, 3, 8), (0.3, 0.5, 0.7),
                                                                              (0.005, 0.01, 0.02)):
                r = evaluate(rows, candidates, accept_fraction, accept_rms)
                sweep.append({"add_fraction": add_fraction, "max_query_fraction": max_query_fraction, "track": tname,
                              "keyframes": keyframes, "candidates": candidates, "accept_inlier_fraction": accept_fraction,
                              "accept_rms": accept_rms, **r})
        summary["sweep"] = sweep
        best = sorted((s for s in sweep if s["false_accepts"] == 0),
                      key=lambda s: (-s["recovered"], s["keyframes"], s["candidates"]))
        summary["sweep_best"] = best[:10]
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(summary, indent=1))
    print(json.dumps({k: v for k, v in summary.items() if k != "sweep"}))


if __name__ == "__main__":
    main()
