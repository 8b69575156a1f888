#!/usr/bin/env python
"""sm_track_frame on the 500-frame VGA bench stream (bench.py's stream: stream_id 0, nominal noise, 5 M surfel cap).

1. Pose-free run: TrackedSession over the whole stream, given only frame 0's pose. Reports the largest and mean
   translational / rotational error against the ground-truth trajectory and the frames reported lost.
2. Timing on the final cloud of the stream integrated with the true poses (sm_stream_run): --timed evenly spaced
   frames are tracked against the cloud (source "cloud") from a guess 1 cm / 0.5 degrees off the true pose, after
   --warmup calls:
     * ms per frame: CUDA events around each call on the caller's stream (the call synchronises once at its end);
     * the split into render (k_render_*), pyramid (bilateral filter, median downscaling) and ICP (k_track_*) from a
       separate pass with sm_profile_kernels (events around every launch, so the parts add up to more than the
       un-profiled time);
     * kernel launches per frame (sm_kernel_launch_count), Gauss-Newton steps applied and the pose error.
Algorithmic bytes of one ICP iteration: per live pixel of the level 2 B of live depth (the four neighbours come from
the same rows) and 16 B of model reads (depth and normal) for an associated pixel.
Prints one JSON summary with the card's name and power limit.
"""
import argparse
import ctypes as C
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
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"


def pose_error(a, b):
    a, b = np.asarray(a, np.float64).reshape(3, 4), np.asarray(b, np.float64).reshape(3, 4)
    Rr = a[:, :3] @ b[:, :3].T   # atan2(sin, cos): acos of the trace alone has a ~0.02 degree floor in fp32
    s = 0.5 * np.linalg.norm([Rr[2, 1] - Rr[1, 2], Rr[0, 2] - Rr[2, 0], Rr[1, 0] - Rr[0, 1]])
    return float(np.linalg.norm(a[:, 3] - b[:, 3])), math.degrees(math.atan2(s, (np.trace(Rr) - 1) / 2))


def perturb(pose, rng):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    angle = math.radians(0.5)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    Rm = np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K
    t = rng.normal(size=3)
    t *= 0.01 / np.linalg.norm(t)
    P = np.asarray(pose, np.float64).reshape(3, 4)
    return np.concatenate([Rm @ P[:, :3], (P[:, 3] + t)[:, None]], axis=1).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--timed", type=int, default=50, help="frames tracked against the final cloud for the timing")
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    product = _lib.load_product()
    cam = S.Camera.tum(640, 480)
    t0 = time.time()
    st = S.make_stream(cam, args.frames, stream_id=0, device="cuda")
    print(f"stream ready in {time.time() - t0:.1f} s", file=sys.stderr)
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    rec = R.CUDASurfelReconstruction(5_000_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)

    # 1. pose-free
    stopped = None
    with R.TrackedSession(rec, pp, ip, st.global_T_frame[0]) as s:
        for f in range(st.frame_count):
            try:
                s.push(st.depth[f], st.color[f])
            except _lib.SurfelError as e:   # a guess that left the fp32 range: report where the run stopped
                stopped = dict(frame=f, error=str(e))
                break
    errors = np.array([pose_error(s.trajectory[f], st.global_T_frame[f]) for f in range(len(s.trajectory))])
    lost = [f for f, r in enumerate(s.results) if not r.tracked]

    # 2. timing against the final cloud of the stream integrated with the true poses
    rec = R.CUDASurfelReconstruction(5_000_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    frames = np.linspace(10, st.frame_count - 10, args.timed).astype(int)
    rng = np.random.RandomState(7)
    guesses = [perturb(st.global_T_frame[f], rng) for f in frames]
    depths = [st.depth[f].cuda() for f in frames]
    for k in range(args.warmup):
        rec.track(depths[k % len(depths)], guesses[k % len(guesses)], pp=pp)
    ms, steps, errs, launches = [], [], [], []
    stream = torch.cuda.current_stream()
    for k, f in enumerate(frames):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        before = product.fn["kernel_launch_count"]()
        a.record(stream)
        pose, res = rec.track(depths[k], guesses[k], pp=pp)
        b.record(stream)
        b.synchronize()
        launches.append(product.fn["kernel_launch_count"]() - before)
        ms.append(a.elapsed_time(b))
        steps.append(res.iterations)
        errs.append(pose_error(pose, st.global_T_frame[f]))
    n = product.fn["profile_kernel_count"]()
    product.fn["profile_kernels"](1)
    product.fn["profile_report"]((C.c_double * n)(), (C.c_uint64 * n)(), n)   # drops earlier records
    for k in range(len(frames)):
        rec.track(depths[k], guesses[k], pp=pp)
    total = (C.c_double * n)()
    count = (C.c_uint64 * n)()
    product.fn["profile_report"](total, count, n)
    product.fn["profile_kernels"](0)
    parts = {"render": 0.0, "pyramid": 0.0, "icp": 0.0}
    per_kernel = {}
    for i in range(n):
        if count[i] == 0:
            continue
        name = product.fn["profile_kernel_name"](i).decode()
        per_kernel[name] = dict(ms_per_frame=total[i] / len(frames), launches_per_frame=count[i] / len(frames))
        part = "render" if name.startswith("k_render") else "icp" if name.startswith("k_track") else "pyramid"
        parts[part] += total[i] / len(frames)
    errs = np.array(errs)
    summary = dict(
        card=card(), frames=int(st.frame_count),
        pose_free=dict(max_translation_mm=float(errors[:, 0].max() * 1000), max_rotation_deg=float(errors[:, 1].max()),
                       mean_translation_mm=float(errors[:, 0].mean() * 1000),
                       mean_rotation_deg=float(errors[:, 1].mean()), lost_frames=lost, stopped=stopped,
                       first_frames=[[round(e[0] * 1000, 3), round(e[1], 4)] for e in errors[:12]]),
        timing=dict(frames=len(frames), ms_median=float(np.median(ms)), ms_p90=float(np.percentile(ms, 90)),
                    launches_per_frame=float(np.median(launches)), steps_median=float(np.median(steps)),
                    profiled_ms_per_frame={k: round(v, 4) for k, v in parts.items()}, per_kernel=per_kernel,
                    max_error_mm=float(errs[:, 0].max() * 1000), max_error_deg=float(errs[:, 1].max())))
    print(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
