"""Cost of --pyramid_level on the GPU: sm_stream_run over a 640x480 synthetic stream at pyramid levels 0, 1 and
2, with device-resident and pinned-host frames, all in one process with the arms alternating.

Prints one JSON line per arm (frames/s over the repeats, h2d_bytes of a run), the mean microseconds of the two
downscaling kernels from sm_profile_kernels in a separate, serialised pass, the per-frame CPU time of the
plain-C restatement (what the reference pays in its upload loop, main.cc:946-981) and the card's name and power
limit. Usage: python tools/pyramid_probe.py [--frames 60] [--repeats 5] [--out DIR]
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

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402
from tests import pyramid_walk  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the name from the runtime at least
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a GPU"
    product = _lib.load_product()
    full = S.Camera.tum(640, 480)
    st = S.make_stream(full, args.frames, stream_id=3, device="cuda")
    torch.cuda.synchronize()
    host = (st.depth.cpu().pin_memory(), st.color.cpu().pin_memory())
    ip = IntegrateParams.defaults()
    first, last = st.integrated_range()
    arms = [(level, on_host) for level in (0, 1, 2) for on_host in (False, True)]
    recs, pps = {}, {}
    for level, on_host in arms:
        cam = full.scaled(level)
        rec = R.CUDASurfelReconstruction(1_500_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
        rec.configure("pyramid_level", level)
        pp = PreprocessParams.defaults()
        pp.depth_valid_region_radius = cam.valid_region_radius()
        recs[(level, on_host)], pps[(level, on_host)] = rec, pp

    def run(arm):
        rec = recs[arm]
        depth, color = host if arm[1] else (st.depth, st.color)
        rec.reset()
        t0 = time.perf_counter()
        s = rec.stream_run(None, depth, color, st.global_T_frame, st.frame_T_global, st.others_TR_reference,
                           pps[arm], ip, first, last)   # returns after a device synchronisation
        return time.perf_counter() - t0, s

    for arm in arms:  # warm-up: graphs, rings, staging
        run(arm)
    times = {arm: [] for arm in arms}
    stats = {}
    for _ in range(args.repeats):
        for arm in arms:
            dt, s = run(arm)
            times[arm].append(dt)
            stats[arm] = s
    info = card()
    results = []
    for arm in arms:
        s = stats[arm]
        fps = [s.frames_integrated / t for t in times[arm]]
        results.append({"pyramid_level": arm[0], "frames_on_host": arm[1], "frames": int(s.frames_integrated),
                        "fps_median": float(np.median(fps)), "fps_min": float(min(fps)), "fps_max": float(max(fps)),
                        "h2d_bytes": int(s.h2d_bytes), "surfels_size": int(s.surfels_size)})

    # kernel times: serialised pass with per-launch events (not part of the frames/s above)
    nk = product.fn["profile_kernel_count"]()
    names = [product.fn["profile_kernel_name"](i).decode() for i in range(nk)]
    tot, cnt = np.zeros(nk), np.zeros(nk, dtype=np.uint64)
    product.call("profile_report", tot.ctypes.data_as(C.POINTER(C.c_double)), cnt.ctypes.data_as(C.POINTER(C.c_uint64)), nk)
    kernels = {}
    for level in (1, 2):
        for on_host in (False, True):
            product.call("profile_kernels", 1)
            run((level, on_host))
            product.call("profile_report", tot.ctypes.data_as(C.POINTER(C.c_double)),
                         cnt.ctypes.data_as(C.POINTER(C.c_uint64)), nk)
            product.call("profile_kernels", 0)
            for name in ("k_downscale_depth_median", "k_downscale_color"):
                i = names.index(name)
                kernels[f"L{level}_{'host' if on_host else 'device'}_{name}"] = {
                    "launches": int(cnt[i]), "mean_us": float(1000.0 * tot[i] / max(int(cnt[i]), 1))}

    # what the reference pays per frame on the CPU: the plain-C restatement, one thread
    depth_np, color_np = st.depth.cpu().numpy(), st.color.cpu().numpy()
    cpu = {}
    for level in (1, 2):
        w, h = 640 >> level, 480 >> level
        pyramid_walk.downscale_median_excluding(depth_np[0], w, h)
        t0 = time.perf_counter()
        n = min(20, args.frames)
        for f in range(n):
            pyramid_walk.downscale_median_excluding(depth_np[f], w, h)
        t1 = time.perf_counter()
        for f in range(n):
            pyramid_walk.color_image_pyramid(color_np[f], level)
        t2 = time.perf_counter()
        cpu[f"L{level}"] = {"depth_ms_per_frame": 1000 * (t1 - t0) / n, "color_ms_per_frame": 1000 * (t2 - t1) / n}

    report = {"card": info, "input": "640x480", "frames": args.frames, "repeats": args.repeats, "runs": results,
              "kernels_profiled": kernels, "cpu_restatement": cpu}
    for r in results:
        print(json.dumps(r))
    print(json.dumps({"kernels_profiled": kernels}))
    print(json.dumps({"cpu_restatement": cpu}))
    print(json.dumps({"card": info}))
    if args.out:
        out = Path(args.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "pyramid_probe.json").write_text(json.dumps(report, indent=1))
    for rec in recs.values():
        rec.close()


if __name__ == "__main__":
    main()
