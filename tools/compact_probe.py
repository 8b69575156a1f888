"""sm_compact (DESIGN.md section 5.13): how much of surfels_size() is merged, what a compaction costs and what it saves.

  * the merged share of surfels_size() every 50 frames along the 500-frame VGA bench stream (5 M cap) and along a
    long synthetic orbit (--orbit-frames at 320 x 240);
  * the time of one sm_compact (CUDA events around the call, median over --calls calls, each on a freshly loaded
    copy of the state) and its kernel split, at the bench's final state and at a synthetic state of --slots slots
    with --merged-fraction of them merged;
  * k_project and whole-frame time (per-kernel events, serial frames) over the last 50 frames of the bench stream,
    continued from the state after frame 450 as it is and after one compaction of it;
  * the device memory the first call allocates.
Prints the card name and power limit read in the same run, and the library version.

    python tools/compact_probe.py [--calls 5] [--orbit-frames 1500] [--slots 4000000] [--out probe_out/compact_probe.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402
from tools.mesh_update_probe import card  # noqa: E402


def kernel_split(lib, fn):
    """Milliseconds per kernel name of everything `fn` launches (per-kernel events, sm_profile_kernels)."""
    lib.fn["profile_kernels"](1)
    fn()
    torch.cuda.synchronize()
    count = lib.fn["profile_kernel_count"]()
    ms, calls = (C.c_double * count)(), (C.c_uint64 * count)()
    lib.fn["profile_report"](ms, calls, count)
    lib.fn["profile_kernels"](0)
    names = [lib.fn["profile_kernel_name"](k).decode() for k in range(count)]
    return {names[k]: round(ms[k], 4) for k in range(count) if calls[k]}


def params(cam):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    return pp, IntegrateParams.defaults()


def make(cam, cap):
    return R.CUDASurfelReconstruction(cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)


def merged_share(cam, st, cap, every=50):
    pp, ip = params(cam)
    rec = make(cam, cap)
    first, last = st.integrated_range()
    out = []
    for a in range(first, last, every):
        b = min(a + every, last)
        rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                       a, b)
        size, live = rec.surfels_size(), rec.surfel_count()
        out.append({"after_frame": b - 1, "surfels_size": size, "merged": size - live,
                    "merged_share": round((size - live) / max(size, 1), 4)})
    return rec, out


def compact_cost(cam, rows, merges, cap, calls):
    lib = _lib.load_product()
    rec = make(cam, cap)
    times = []
    stats = None
    for i in range(calls):
        rec.load_state(rows, merges)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        stats = rec.compact()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    rec.load_state(rows, merges)
    split = kernel_split(lib, lambda: rec.compact())
    return {"slots_before": int(stats.slots_before), "slots_after": int(stats.slots_after),
            "links_dropped": int(stats.links_dropped), "median_ms": round(float(np.median(times)), 3),
            "min_ms": round(float(np.min(times)), 3), "kernel_split_ms": split}


def frame_times(cam, st, rows, merges, cap, compact, first, last):
    lib = _lib.load_product()
    pp, ip = params(cam)
    rec = make(cam, cap)
    rec.load_state(rows, merges)
    if compact:
        rec.compact()
    size_at_start = rec.surfels_size()
    rec.enable_timings(True)   # serial frames: per-kernel events are meaningful
    split = kernel_split(lib, lambda: rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global,
                                                     st.others_TR_reference, pp, ip, first, last))
    frames = last - first
    total = sum(split.values())
    return {"surfels_size_at_start": int(size_at_start),
            "k_project_ms_per_frame": round(split.get("k_project", 0.0) / frames, 4),
            "kernel_ms_per_frame": round(total / frames, 4)}


def synthetic_state(n, merged_fraction, seed=1):
    rng = np.random.default_rng(seed)
    rows = rng.random((_lib.ROW_COUNT, n), dtype=np.float32)
    rows[18] = np.zeros(n, np.uint32).view(np.float32)   # stamps below 2^31
    merged = rng.random(n) < merged_fraction
    rows[7, merged] = -1.0
    links = rng.integers(0, n, size=(4, n), dtype=np.uint32)
    rows[19:23] = links.view(np.float32)
    rows[24] = np.zeros(n, np.uint32).view(np.float32)
    return rows, int(merged.sum())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--orbit-frames", type=int, default=1500)
    ap.add_argument("--slots", type=int, default=4_000_000)
    ap.add_argument("--merged-fraction", type=float, default=0.3)
    ap.add_argument("--out", type=Path, default=Path("probe_out/compact_probe.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    result = {"card": card(), "build": _lib.load_product().version()}

    vga = S.Camera.tum(640, 480)
    st = S.make_stream(vga, 500, device="cuda")
    rec, result["bench_stream_merged_share"] = merged_share(vga, st, 5_000_000)
    rows, n, merges = rec.dump_state()
    rec.close()
    result["bench_final_compact"] = compact_cost(vga, rows, merges, 5_000_000, args.calls)

    # k_project / frame time over the last 50 frames, continued from the state after frame 450
    pp, ip = params(vga)
    base = make(vga, 5_000_000)
    first, last = st.integrated_range()
    base.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                    first, last - 46)
    rows450, _, merges450 = base.dump_state()
    base.close()
    result["frames_after_450"] = {
        "uncompacted": frame_times(vga, st, rows450, merges450, 5_000_000, False, last - 46, last),
        "compacted": frame_times(vga, st, rows450, merges450, 5_000_000, True, last - 46, last)}
    del st
    torch.cuda.empty_cache()

    qvga = S.Camera.tum(320, 240)
    orbit = S.make_stream(qvga, args.orbit_frames, device="cuda")
    rec, result["orbit_merged_share"] = merged_share(qvga, orbit, 5_000_000, every=100)
    rec.close()
    del orbit
    torch.cuda.empty_cache()

    srows, smerged = synthetic_state(args.slots, args.merged_fraction)
    result["synthetic_compact"] = compact_cost(qvga, srows, smerged, args.slots + 1024, args.calls)

    # memory of the first call that removes something, at the bench cap
    mem = make(vga, 5_000_000)
    mem.load_state(rows, merges)
    torch.cuda.synchronize()
    free_before = torch.cuda.mem_get_info()[0]
    mem.compact()
    torch.cuda.synchronize()
    result["first_call_allocates_bytes_at_5M_cap"] = int(free_before - torch.cuda.mem_get_info()[0])

    text = json.dumps(result, indent=1)
    print(text)
    args.out.parent.mkdir(parents=True, exist_ok=True)
    args.out.write_text(text)


if __name__ == "__main__":
    main()
