#!/usr/bin/env python
"""Incremental sessions against sm_stream_run on the 500-frame VGA bench stream (bench.py's stream, stream_id 0).

Arms, alternating within one run:
  stream_run   sm_stream_run over device frames (bench.py's flagship path)
  session      a session fed device frames, one push per frame
  session_host a session fed pageable host frames (numpy arrays)
  session_xfer a session fed device frames, with sm_transfer_delta_to_cpu into persistent buffers every 10 frames
  per_frame    sm_preprocess + sm_integrate per frame, the path of a caller without sessions
Prints one JSON object with the card's name and power limit, and frames/s (integrated frames over the
synchronised wall time) and host milliseconds per push (or per frame) of every run.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, TransferToken  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cap", type=int, default=5_000_000)
    ap.add_argument("--arms", default="stream_run,session,session_host,session_xfer,per_frame")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cam = S.Camera.tum(640, 480)
    st = S.make_stream(cam, args.frames, stream_id=0, device="cuda")
    K = 8
    others = R.stream_outlier_filter_transforms(st.global_T_frame, st.frame_T_global, K, st.depth_scaling)
    host_depth, host_color = st.depth.cpu().numpy(), st.color.cpu().numpy()
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    rec = R.CUDASurfelReconstruction(args.cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    F, half = args.frames, K // 2
    out_depth = torch.zeros((cam.height, cam.width), dtype=torch.uint16, device="cuda")
    out_normals = torch.zeros((cam.height, cam.width, 2), dtype=torch.float32, device="cuda")
    out_radius = torch.zeros((cam.height, cam.width), dtype=torch.float32, device="cuda")
    xfer_bufs = R.make_cpu_buffers(args.cap)

    def arm_stream_run():
        stats = rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, others, pp, ip, half,
                               F - half)
        return stats.frames_integrated, stats.host_enqueue_ms / F

    def arm_session(source, transfer=False):
        host = 0.0
        token = TransferToken()
        with rec.session(pp, ip, (cam.width, cam.height)) as s:
            for f in range(F):
                d, c = (st.depth[f], st.color[f]) if source == "device" else (host_depth[f], host_color[f])
                t = time.perf_counter()
                status = s.push(d, c, st.global_T_frame[f], st.frame_T_global[f])
                host += time.perf_counter() - t
                if transfer and f % 10 == 9:
                    rec.TransferDeltaToCPU(None, status.last_integrated_frame, xfer_bufs, token)
        return s.stats.frames_integrated, host * 1e3 / F

    def arm_per_frame():
        host = 0.0
        for f in range(half, F - half):
            t = time.perf_counter()
            rec.preprocess(None, pp, st.depth[f], [st.depth[o] for o in S_others(f, K)], others[f], out_depth,
                           out_normals, out_radius)
            rec.integrate(None, f, ip, out_depth, out_normals, out_radius, st.color[f], st.global_T_frame[f],
                          st.frame_T_global[f])
            host += time.perf_counter() - t
        return F - 2 * half, host * 1e3 / (F - 2 * half)

    arms = {"stream_run": arm_stream_run, "session": lambda: arm_session("device"),
            "session_host": lambda: arm_session("host"), "session_xfer": lambda: arm_session("device", True),
            "per_frame": arm_per_frame}
    selected = [a for a in args.arms.split(",") if a]
    results = {a: [] for a in selected}
    for name in selected:   # warm-up: graph instantiation, rings, staging
        rec.reset()
        arms[name]()
    torch.cuda.synchronize()
    for rep in range(args.reps):
        for name in selected:
            rec.reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            frames, host_ms = arms[name]()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            rec_count = rec.surfels_size()
            results[name].append({"fps": frames / wall, "host_ms_per_push": host_ms, "surfels_size": rec_count})
            print(f"rep {rep} {name:13s} {frames / wall:8.1f} frames/s  host {host_ms:.4f} ms/push  "
                  f"surfels {rec_count}", flush=True)
    summary = {"card": card(), "frames": F, "reps": args.reps,
               "arms": {a: {"fps_median": float(np.median([r["fps"] for r in v])),
                            "fps_min": float(min(r["fps"] for r in v)), "fps_max": float(max(r["fps"] for r in v)),
                            "host_ms_per_push_median": float(np.median([r["host_ms_per_push"] for r in v]))}
                        for a, v in results.items()}}
    print(json.dumps(summary))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(summary, indent=1))


def S_others(frame, K):
    half = K // 2
    return [frame - (i + 1) for i in range(half)] + [frame + (i + 1) for i in range(half)]


if __name__ == "__main__":
    main()
