#!/usr/bin/env python
"""Same-box A/B of builds of the product library (run on a GPU): one synthetic stream, one process, the
product first and last and every --lib name=path build in between (a variant is built with
`python -m surfelmeshing_b200.build --out variants/lib_<name>.so -- <nvcc flags>`). Prints frames/s (best and
median of --reps passes, CUDA events) and the surfel counts; writes probe_out/ab_probe.json."""
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


def load_build(path):
    """Another build of the product library, bound to the entry points it exports: an older build (the parent
    commit's) may lack ones added since, and the A/B only calls the ones both have."""
    lib = _lib.Library.__new__(_lib.Library)
    lib.path, lib.prefix, lib.cdll, lib.fn = Path(path).resolve(), "sm_", C.CDLL(str(Path(path).resolve()), mode=C.RTLD_LOCAL), {}
    for name, (restype, argtypes) in {**_lib._SIGNATURES, **_lib._PRODUCT_ONLY}.items():
        f = getattr(lib.cdll, "sm_" + name, None)
        if f is not None:
            f.restype, f.argtypes = restype, argtypes
            lib.fn[name] = f
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--cap", type=int, default=5_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host", action="store_true", help="pinned host frames (e2e path)")
    ap.add_argument("--sigma-xy", type=float, default=None,
                    help="bilateral_filter_sigma_xy (default 3: radius 6, the fused kernel; 2 gives radius 4)")
    ap.add_argument("--lib", action="append", default=[],
                    help="name=path of another product build; the product itself runs first and last")
    ap.add_argument("--out", default="probe_out/ab_probe.json")
    args = ap.parse_args()

    product = _lib.load_product()
    arms = [("default", product)]
    for item in args.lib:
        name, path = item.split("=", 1)
        arms.append((name, load_build(path)))
    arms.append(("default_again", product))

    cam = S.Camera.tum(args.width, args.height)
    st = S.make_stream(cam, args.frames, device="cuda")
    depth, color = st.depth, st.color
    if args.host:
        depth, color = depth.cpu().pin_memory(), color.cpu().pin_memory()
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    if args.sigma_xy is not None:
        pp.bilateral_filter_sigma_xy = args.sigma_xy
    ip = IntegrateParams.defaults()
    f0, f1 = st.integrated_range()
    torch.cuda.synchronize()
    results = []
    for name, lib in arms:
        rec = R.CUDASurfelReconstruction(args.cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=lib)
        rates, host_ms = [], []
        stats = None
        for rep in range(args.reps + 1):  # first pass = warm-up (graph instantiation, buffers)
            rec.reset()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            stats = rec.stream_run(None, depth, color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                                   ip, f0, f1)
            e1.record()
            torch.cuda.synchronize()
            if rep:
                rates.append(stats.frames_integrated / e0.elapsed_time(e1) * 1e3)
                host_ms.append(stats.host_enqueue_ms)
        rec.close()
        entry = {"config": name, "lib": str(lib.path), "fps_best": max(rates), "fps_median": float(np.median(rates)),
                 "host_enqueue_ms": float(np.median(host_ms)), "surfels_size": int(stats.surfels_size),
                 "surfel_count": int(stats.surfel_count), "launches": int(stats.kernel_launches)}
        results.append(entry)
        print(f"{name:28s} best {entry['fps_best']:9.1f}  median {entry['fps_median']:9.1f} fps   host enqueue "
              f"{entry['host_enqueue_ms']:7.2f} ms   surfels {entry['surfels_size']} / {entry['surfel_count']}  "
              f"launches {entry['launches']}", flush=True)
    Path(args.out).parent.mkdir(exist_ok=True)
    Path(args.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
