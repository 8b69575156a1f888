"""sm_mesh_fill_holes on the final cloud of the 500-frame VGA synthetic stream (the bench workload): the stats at
K = 4, 8 and 16, the time of one call with enough capacity (median and p90 over synchronised calls, CUDA events
around the call) next to sm_triangulate's on the same mesh, and the kernel split of one such call; and on golden f7
the area of mesh and fill against the reference's CPU mesher (oracle/meshing_ref.py, when built). Prints the card
name and power limit read in the same run.

    python tools/mesh_holes_probe.py [--frames 500] [--calls 20] [--out probe_out/mesh_holes_probe.json]
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
from surfelmeshing_b200._lib import HoleParams, IntegrateParams, PreprocessParams  # noqa: E402
from tools.mesh_update_probe import card  # noqa: E402


def event_ms(fn, calls):
    fn()
    times = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return {"median_ms": round(float(np.median(times)), 4), "p90_ms": round(float(np.percentile(times, 90)), 4)}


def kernel_split(lib, fn):
    lib.fn["profile_kernels"](1)
    fn()
    torch.cuda.synchronize()
    count = lib.fn["profile_kernel_count"]()
    ms, calls = (C.c_double * count)(), (C.c_uint64 * count)()
    lib.fn["profile_report"](ms, calls, count)
    lib.fn["profile_kernels"](0)
    names = [lib.fn["profile_kernel_name"](k).decode() for k in range(count)]
    return {names[k]: round(ms[k], 4) for k in range(count) if calls[k] and names[k].startswith(("k_hole", "k_reg_mirror"))}


def reference_area():
    from oracle import meshing_ref
    from tests import hole_walk as HW, mesh_walk as M
    rows = M.golden_f7()
    tri, _, _ = M.triangulate(rows)
    if not meshing_ref.available():
        return {"reference": "not built"}
    ref = meshing_ref.SurfelMeshing()
    ref.integrate(1, *[rows[k] for k in (3, 4, 5, 7, 8, 9, 10)], rows[18].view(np.uint32))
    ref.check_remeshing()
    ref.triangulate()
    ref_area = M.area(rows, ref.triangles())
    ref.close()
    out = {"mesh": round(M.area(rows, tri) / ref_area, 4)}
    for K in (4, 8, 16):
        f, _ = HW.fill_holes(rows, tri, HoleParams(K, 90.0, 180.0))
        out[f"K={K}"] = round(M.area(rows, np.concatenate([tri, f]).astype(np.int64)) / ref_area, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--calls", type=int, default=20)
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
    tri, mesh_stats = rec.triangulate()
    result = {"card": card(), "surfels_size": rec.surfels_size(), "triangles": len(tri),
              "triangulate": event_ms(rec.triangulate, args.calls), "fill": {}}
    for K in (4, 8, 16):
        p = HoleParams(K, 90.0, 180.0)
        fill, stats = rec.fill_holes(tri, p)
        entry = {k: int(getattr(stats, k)) for k, _ in _lib.HoleStats._fields_}
        # One sm_mesh_fill_holes call into a buffer that is large enough (fill_holes() makes a count query first).
        out = torch.empty((max(len(fill), 1), 3), dtype=torch.int32, device="cuda")
        direct_stats = _lib.HoleStats()

        def direct():
            lib.call("mesh_fill_holes", rec._h, None, C.byref(p), C.c_void_p(tri.data_ptr()), len(tri),
                     C.c_void_p(out.data_ptr()), len(out), C.byref(direct_stats))

        entry.update(event_ms(direct, args.calls))
        entry["kernel_ms"] = kernel_split(lib, direct)
        result["fill"][f"K={K}"] = entry
    rec.close()
    result["golden_f7_area_vs_reference"] = reference_area()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text)


if __name__ == "__main__":
    main()
