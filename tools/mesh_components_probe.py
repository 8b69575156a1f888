"""sm_mesh_components on the final cloud of the 500-frame VGA synthetic stream (the bench workload) and of the same
stream with twice its depth noise, each meshed by sm_triangulate with the holes of up to 8 edges filled: the pieces
and a histogram of their sizes and areas; the share of triangles and area in pieces below several size thresholds;
the time of one call (median and p90 over synchronised calls, CUDA events around the call) next to
sm_triangulate's; the kernel split of one call (torch.profiler); and, for the full mesh and the mesh filtered at
several settings, the covered pixels and the depth error (median / p95) of sm_render_mesh against the ray-cast scene
from three of the stream's cameras. Prints the card name and power limit read in the same run.

    python tools/mesh_components_probe.py [--frames 500] [--calls 10] [--out probe_out/mesh_components_probe.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import re
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import ComponentParams, HoleParams, IntegrateParams, PreprocessParams  # noqa: E402
from tools.mesh_holes_probe import event_ms  # noqa: E402
from tools.mesh_simplify_probe import depth_error  # noqa: E402
from tools.mesh_update_probe import card  # noqa: E402

SIZE_THRESHOLDS = (2, 5, 10, 20, 50, 100, 1000)
SETTINGS = {"min_triangles 5": ComponentParams.defaults(min_triangles=5),
            "min_triangles 10 (default)": ComponentParams.defaults(),
            "min_triangles 20": ComponentParams.defaults(min_triangles=20),
            "min_triangles 50": ComponentParams.defaults(min_triangles=50),
            "min_area 1e-4 m^2": ComponentParams.defaults(min_triangles=0, min_area=1e-4),
            "keep_largest 1": ComponentParams.defaults(min_triangles=0, keep_largest=1)}


def kernel_split(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"k_cc_\w+|k_knn_scan_\w+|DeviceRadixSort\w+", e.key)
        if m:
            name = m.group(0)
            ms = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
            prev = out.get(name, [0.0, 0])
            out[name] = [round(prev[0] + ms, 4), prev[1] + int(e.count)]
    return out


def probe(lib, name, noise_scale, frames, calls):
    cam = S.Camera.tum(640, 480)
    st = S.make_stream(cam, frames, device="cuda", noise_scale=noise_scale)
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    rec = R.CUDASurfelReconstruction(5_000_000, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                   IntegrateParams.defaults(), first, last)
    tri, _ = rec.triangulate()
    fill, _ = rec.fill_holes(tri, HoleParams(8, 90.0, 180.0))
    mesh = torch.cat([tri, fill])
    views = (first + 10, (first + last) // 2, last - 4)
    _, labels, table, stats = rec.mesh_components(mesh, ComponentParams.defaults(min_triangles=0))
    sizes = table["triangles"].cpu().numpy()
    area = table["area"].cpu().numpy()
    T, A = int(sizes.sum()), float(area.sum())
    result = {"stream": name, "surfels_size": rec.surfels_size(), "triangles": T, "area_m2": round(A, 4),
              "pieces": int(stats.components), "largest": [int(stats.largest_triangles), round(stats.largest_area, 4)],
              "ten_largest": sorted(sizes.tolist(), reverse=True)[:10], "below": {}}
    edges = [1, 2, 5, 10, 20, 50, 100, 1000, 10000, 10 ** 9]
    # pieces, triangles and area (m^2) per size bin
    result["size_histogram"] = {f"[{lo}, {hi})": [int(((sizes >= lo) & (sizes < hi)).sum()),
                                                  int(sizes[(sizes >= lo) & (sizes < hi)].sum()),
                                                  round(float(area[(sizes >= lo) & (sizes < hi)].sum()), 5)]
                                for lo, hi in zip(edges[:-1], edges[1:])}
    area_edges = [0, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e-1, 1.0, 1e9]
    result["area_histogram_m2"] = {f"[{lo:g}, {hi:g})": int(((area >= lo) & (area < hi)).sum())
                                   for lo, hi in zip(area_edges[:-1], area_edges[1:])}
    for b in SIZE_THRESHOLDS:
        small = sizes < b
        result["below"][f"< {b} triangles"] = {"pieces": int(small.sum()), "triangle_share": round(sizes[small].sum() / T, 6),
                                               "area_share": round(float(area[small].sum()) / A, 6)}
    out = torch.empty((len(mesh), 3), dtype=torch.int32, device="cuda")
    lab = torch.empty(len(mesh), dtype=torch.int32, device="cuda")
    raw = torch.empty((len(mesh), C.sizeof(_lib.MeshComponent)), dtype=torch.uint8, device="cuda")
    p = ComponentParams.defaults()
    s = _lib.ComponentStats()

    def direct():
        lib.call("mesh_components", rec._h, None, C.byref(p), C.c_void_p(mesh.data_ptr()), len(mesh),
                 C.c_void_p(out.data_ptr()), len(out), C.c_void_p(lab.data_ptr()), C.c_void_p(raw.data_ptr()),
                 len(mesh), C.byref(s))

    result["triangulate"] = event_ms(rec.triangulate, calls)
    result["components_call"] = event_ms(direct, calls)
    result["kernel_ms"] = kernel_split(direct)
    full = depth_error(rec, cam, st, mesh, views)
    result["depth_error"] = {"full": full}
    for label, q in SETTINGS.items():
        kept, _, _, ks = rec.mesh_components(mesh, q)
        e = depth_error(rec, cam, st, kept, views)
        e["covered_share"] = round(e["covered_px"] / max(full["covered_px"], 1), 6)
        e["triangles_out"] = int(ks.triangles_out)
        e["components_kept"] = int(ks.components_kept)
        result["depth_error"][label] = e
    print(json.dumps(result), flush=True)
    rec.close()
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    lib = _lib.load_product()
    result = {"card": card(), "streams": [probe(lib, "bench", 1.0, args.frames, args.calls),
                                          probe(lib, "bench, depth noise x 2", 2.0, args.frames, args.calls)]}
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text)


if __name__ == "__main__":
    main()
