"""sm_mesh_update along the 500-frame VGA synthetic stream (the bench workload) pushed through a session, with an
update after every push: the time of each update (host clock around the synchronous call), |C|/n, |A|/n, |R|/n
and the delta sizes, sm_triangulate's time on the same states at a few frames, the session's frames/s with and
without the updates, and on the final cloud a sparse case (1 000 slots nudged) and a sweep of change fractions
with the kernel split, from which the list / sweep threshold of k_mesh_umbrella_update is read. Prints the card
name and power limit read in the same run.

    python tools/mesh_update_probe.py [--frames 500] [--out probe_out/mesh_update_probe.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = f"unavailable ({e})"
    return out or torch.cuda.get_device_name(0)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def triangulate_ms(rec, calls=5):
    rec.triangulate()
    return float(np.median([timed(rec.triangulate)[0] for _ in range(calls)]))


def row(st, n, ms):
    return {"ms": round(ms, 3), "n": n, "C": int(st.slots_changed), "A": int(st.umbrellas_rebuilt),
            "R": int(st.owners_rechecked), "C/n": st.slots_changed / max(n, 1), "A/n": st.umbrellas_rebuilt / max(n, 1),
            "R/n": st.owners_rechecked / max(n, 1), "added": int(st.triangles_added),
            "removed": int(st.triangles_removed), "triangles": int(st.mesh.triangle_count),
            "full_sweep": int(st.full_sweep)}


def warm_transition(replay, before, after, calls=3):
    """The update from state `before` to state `after` and sm_triangulate on `after`, both on a handle whose buffers
    already fit (median of `calls`): what a call costs once the first call at that size has grown the buffers."""
    update = []
    for _ in range(calls):
        replay.load_state(*before)
        replay.mesh_update()
        replay.load_state(*after)
        update.append(timed(replay.mesh_update)[0])
    return float(np.median(update)), triangulate_ms(replay)


def session(st, cam, pp, update, checkpoints=()):
    rec = R.CUDASurfelReconstruction(5_000_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    replay = R.CUDASurfelReconstruction(5_000_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    rows, tri_ms, warm, before = [], {}, {}, None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with rec.session(pp, IntegrateParams.defaults(), (cam.width, cam.height)) as s:
        for k in range(st.frame_count):
            s.push(st.depth[k], st.color[k], st.global_T_frame[k], st.frame_T_global[k])
            if update:
                ms, u = timed(rec.mesh_update)
                rows.append(row(u, rec.surfels_size(), ms))
                if k + 1 in checkpoints:
                    tri_ms[k + 1] = triangulate_ms(rec)
                    state, _, merges = rec.dump_state()
                    warm[k + 1] = warm_transition(replay, before, (state, merges))
                if k + 2 in checkpoints:
                    state, _, merges = rec.dump_state()
                    before = (state, merges)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    replay.close()
    return rec, rows, tri_ms, warm, st.frame_count / seconds


def kernel_split(lib, fn):
    lib.fn["profile_kernels"](1)
    out = fn()
    torch.cuda.synchronize()
    count = lib.fn["profile_kernel_count"]()
    ms = (C.c_double * count)()
    calls = (C.c_uint64 * count)()
    lib.fn["profile_report"](ms, calls, count)
    lib.fn["profile_kernels"](0)
    split = {lib.fn["profile_kernel_name"](k).decode(): round(ms[k], 4) for k in range(count)
             if calls[k] and lib.fn["profile_kernel_name"](k).decode().startswith(("k_mesh", "k_reg_mirror"))}
    return out, split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    lib = _lib.load_product()
    cam = S.Camera.tum(640, 480)
    st = S.make_stream(cam, args.frames, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    checkpoints = sorted({min(100, args.frames), min(250, args.frames), args.frames})

    plain, _, _, _, fps_plain = session(st, cam, pp, update=False)
    plain.close()
    rec, rows, tri_ms, warm, fps_update = session(st, cam, pp, update=True, checkpoints=checkpoints)
    steady = [r["ms"] for r in rows[20:]] or [r["ms"] for r in rows]
    result = {
        "card": card(), "frames": args.frames,
        "update_ms_median": float(np.median(steady)), "update_ms_p90": float(np.percentile(steady, 90)),
        "session_fps_without_update": fps_plain, "session_fps_with_update": fps_update,
        # in the session (the first call at a size also grows the buffers), and the same transition replayed on a
        # handle whose buffers fit, against sm_triangulate on that handle
        "at_frames": {str(k): {**rows[k - 1], "triangulate_ms": tri_ms.get(k), "warm_update_ms": warm[k][0],
                               "warm_triangulate_ms": warm[k][1]} for k in checkpoints},
        "full_sweeps": sum(r["full_sweep"] for r in rows),
        "share_A_over_n": {q: float(np.percentile([r["A/n"] for r in rows[20:] or rows], q)) for q in (10, 50, 90)},
    }

    # the final cloud: no change, 1 000 slots nudged, then growing change fractions with the kernel split
    state, n, merges = rec.dump_state()
    rng = np.random.default_rng(0)
    present = np.flatnonzero(state[7] > 0)
    result["final_triangulate_ms"] = triangulate_ms(rec)
    rec.mesh_update()   # (sm_session_end integrated the last frames)
    result["final_no_change_ms"] = timed(rec.mesh_update)[0]
    fractions = {}
    for label, count in [("sparse_1000", 1000)] + [(f"nudge_{f}", int(f * len(present)))
                                                    for f in (0.002, 0.005, 0.01, 0.02, 0.05, 0.1, 0.3)]:
        rec.load_state(state, merges)
        rec.mesh_update()
        edited = state.copy()
        pick = rng.choice(present, count, replace=False)
        edited[3, pick] = np.nextafter(edited[3, pick], np.float32(np.inf))
        rec.load_state(edited, merges)
        ms, u = timed(rec.mesh_update)
        entry = row(u, n, ms)
        rec.load_state(state, merges)
        rec.mesh_update()
        rec.load_state(edited, merges)
        entry["warm_ms"] = timed(rec.mesh_update)[0]   # the same update again, its buffers already grown
        rec.load_state(state, merges)
        rec.mesh_update()
        rec.load_state(edited, merges)
        _, split = kernel_split(lib, rec.mesh_update)
        entry["kernel_ms"] = split
        fractions[label] = entry
    result["final_cloud"] = fractions
    print(json.dumps(result))
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(result, indent=1))
    rec.close()


if __name__ == "__main__":
    main()
