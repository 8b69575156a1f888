#!/usr/bin/env python
"""Device timeline of the frame pipeline (sm_timeline_enable): per-kernel start/end stamps
written by the kernels themselves while sm_stream_run pipelines the stream (or, with --session, while a session
is pushed the same frames from device memory). Prints the mean duration per kernel, the frame period, the time
per frame in which no kernel of the pipeline runs, and a few consecutive frames as a Gantt table; writes the
raw stamps to probe_out/timeline.csv."""
import argparse
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--show", type=int, default=450, help="first frame of the Gantt table")
    ap.add_argument("--count", type=int, default=3)
    ap.add_argument("--out", default="probe_out/timeline.csv")
    ap.add_argument("--session", action="store_true", help="push the frames through a session instead")
    args = ap.parse_args()
    lib = _lib.load_product()
    cam = S.Camera.tum(640, 480)
    st = S.make_stream(cam, args.frames, device="cuda")
    depth, color = st.depth.cuda(), st.color.cuda()
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    f0, f1 = st.integrated_range()
    rec = R.CUDASurfelReconstruction(5_000_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=lib)
    n_frames = 1 << (args.frames - 1).bit_length()
    for rep in range(2):
        rec.reset()
        if rep == 1:
            lib.call("timeline_enable", rec._h, n_frames)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if args.session:
            with rec.session(pp, ip, (cam.width, cam.height)) as s:
                for f in range(args.frames):
                    s.push(depth[f], color[f], st.global_T_frame[f], st.frame_T_global[f])
            stats = s.stats
        else:
            stats = rec.stream_run(None, depth, color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                                   ip, f0, f1)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        print(f"rep {rep}: {stats.frames_integrated} frames {ms:.2f} ms -> {stats.frames_integrated / ms * 1e3:.1f} fps")
    kcount = lib.fn["profile_kernel_count"]()
    names = [lib.fn["profile_kernel_name"](i).decode() for i in range(kcount)]
    buf = np.zeros((n_frames, kcount, 2), dtype=np.uint64)
    lib.call("timeline_read", rec._h, buf.ctypes.data_as(C.POINTER(C.c_uint64)), n_frames)
    valid = buf[:, :, 0] != np.uint64(0xFFFFFFFFFFFFFFFF)
    start = buf[:, :, 0].astype(np.float64)
    end = buf[:, :, 1].astype(np.float64)
    Path(args.out).parent.mkdir(exist_ok=True)
    with open(args.out, "w") as fh:
        fh.write("frame,kernel,start_ns,end_ns\n")
        for f in range(n_frames):
            for k in range(kcount):
                if valid[f, k]:
                    fh.write(f"{f},{names[k]},{int(buf[f, k, 0])},{int(buf[f, k, 1])}\n")
    lo, hi = f0 + 100, f1 - 10
    print(f"mean over frames {lo}..{hi} (us):")
    for k in range(kcount):
        v = valid[lo:hi, k]
        if v.any():
            d = (end[lo:hi, k] - start[lo:hi, k])[v] / 1e3
            print(f"  {names[k]:28s} {d.mean():7.2f}  (min {d.min():6.2f} max {d.max():6.2f})")
    kp = names.index("k_project")
    period = np.diff(start[lo:hi, kp]) / 1e3
    print(f"frame period (project start to project start): mean {period.mean():.2f} us  median {np.median(period):.2f}")
    # device time without any pipeline kernel running, between the first kernel of frame lo and frame hi's k_project
    w0, w1 = start[lo][valid[lo]].min(), start[hi, kp]
    spans = sorted((s_, e_) for f in range(lo - 3, hi + 3) for s_, e_, ok in zip(start[f], end[f], valid[f])
                   if ok and e_ > w0 and s_ < w1)
    idle, cursor = 0.0, w0
    for s_, e_ in spans:
        if s_ > cursor:
            idle += s_ - cursor
        cursor = max(cursor, e_)
    idle += max(0.0, w1 - cursor)
    print(f"no pipeline kernel running: {idle / 1e3 / (hi - lo):.2f} us per frame")
    t0 = start[args.show, kp]
    for f in range(args.show, args.show + args.count):
        rows = [(start[f, k], end[f, k], names[k]) for k in range(kcount) if valid[f, k]]
        print(f"frame {f}:")
        for s_, e_, n_ in sorted(rows):
            print(f"  {n_:28s} {(s_ - t0) / 1e3:8.2f} -> {(e_ - t0) / 1e3:8.2f}  ({(e_ - s_) / 1e3:6.2f})")


if __name__ == "__main__":
    main()
