"""sm_triangulate on the final cloud of the 500-frame VGA synthetic stream (the bench workload): time per call
(CUDA events around synchronised calls after warm-up), a kernel split from a separate profiled pass, the mesh
statistics, and - where oracle/_ref/libmeshing_ref.so is built - the reference's CPU Triangulate() on the same
cloud. Prints the card name and power limit read in the same run.

    python tools/mesh_probe.py [--frames 500] [--calls 20] [--ref-slots 60000] [--out probe_out/mesh_probe.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--ref-slots", type=int, default=60000, help="largest cloud the CPU mesher is given")
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    lib = _lib.load_product()
    cam = S.Camera.tum(640, 480)
    st = S.make_stream(cam, args.frames, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    rec = R.CUDASurfelReconstruction(5_000_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                   IntegrateParams.defaults(), first, last)
    n = rec.surfels_size()
    for _ in range(3):
        tri, stats = rec.triangulate()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        tri, stats = rec.triangulate()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    lib.fn["profile_kernels"](1)
    rec.triangulate()
    torch.cuda.synchronize()
    count = lib.fn["profile_kernel_count"]()
    ms = (C.c_double * count)()
    calls = (C.c_uint64 * count)()
    lib.fn["profile_report"](ms, calls, count)
    lib.fn["profile_kernels"](0)
    split = {lib.fn["profile_kernel_name"](k).decode(): round(ms[k], 4) for k in range(count)
             if calls[k] and lib.fn["profile_kernel_name"](k).decode().startswith(("k_mesh", "k_reg_mirror"))}
    result = {
        "card": card(), "surfels_size": n, "calls": args.calls,
        "median_ms": float(np.median(times)), "p90_ms": float(np.percentile(times, 90)),
        "kernel_ms": split,
        "triangles": int(stats.triangle_count), "vertices_meshed": int(stats.vertices_meshed),
        "boundary_edges": int(stats.boundary_edges), "umbrella_overflows": int(stats.umbrella_overflows),
    }
    from oracle import meshing_ref
    if meshing_ref.available():
        rows, n_all, _ = rec.dump_state()
        take = min(n_all, args.ref_slots)
        sub = rows[:, :take]
        ref = meshing_ref.SurfelMeshing()
        t0 = time.perf_counter()
        ref.integrate(1, *[sub[k] for k in (3, 4, 5, 7, 8, 9, 10)], sub[18].view(np.uint32))
        ref.check_remeshing()
        ref.triangulate()
        t1 = time.perf_counter()
        small = R.CUDASurfelReconstruction(max(take, 1024), cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
        small.load_state(sub, 0)
        tri_small, st_small = small.triangulate()
        result["reference_cpu"] = {"slots": take, "seconds": t1 - t0, "triangles": len(ref.triangles()),
                                   "gpu_triangles_same_cloud": int(st_small.triangle_count)}
        ref.close()
        small.close()
    print(json.dumps(result))
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(result, indent=1))
    rec.close()


if __name__ == "__main__":
    main()
