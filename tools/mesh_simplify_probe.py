"""sm_mesh_simplify on the final cloud of the 500-frame VGA synthetic stream (the bench workload), meshed by
sm_triangulate with the holes of up to 8 edges filled: triangles and vertices out at targets of 50, 25 and 10 % (no
cost bound) and with the default max_cost alone; rounds and collapses per round; the time of one call (median and
p90 over synchronised calls, CUDA events around the call) next to sm_triangulate's on the same cloud; the kernel
split of one call; and the depth error of the rendered meshes against the ray-cast scene from three of the stream's
cameras. Prints the card name and power limit read in the same run.

    python tools/mesh_simplify_probe.py [--frames 500] [--calls 10] [--out probe_out/mesh_simplify_probe.json]
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
from surfelmeshing_b200._lib import HoleParams, IntegrateParams, PreprocessParams, SimplifyParams  # noqa: E402
from tools.mesh_holes_probe import event_ms  # noqa: E402
from tools.mesh_update_probe import card  # noqa: E402


def kernel_split(lib, fn):
    lib.fn["profile_kernels"](1)
    fn()
    torch.cuda.synchronize()
    count = lib.fn["profile_kernel_count"]()
    ms, calls = (C.c_double * count)(), (C.c_uint64 * count)()
    lib.fn["profile_report"](ms, calls, count)
    lib.fn["profile_kernels"](0)
    names = [lib.fn["profile_kernel_name"](k).decode() for k in range(count)]
    return {names[k]: [round(ms[k], 4), int(calls[k])] for k in range(count)
            if calls[k] and names[k].startswith(("k_simplify", "k_reg_mirror"))}


def depth_error(rec, cam, st, tri, frames):
    view = dict(width=cam.width, height=cam.height, fx=cam.fx, fy=cam.fy, cx=cam.cx, cy=cam.cy, near=0.1, far=20.0,
                unmeshed_surfels=False, outputs=("depth",))
    poses = S.trajectory(st.frame_count)
    errs, covered = [], 0
    for f in frames:
        gt, _ = S._raycast(cam, torch.from_numpy(poses[f]).to("cuda"), "cuda")
        d = rec.render_mesh(tri, st.frame_T_global[f], **view)["depth"].double()
        mask = (d > 0) & torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0)
        covered += int(mask.sum())
        errs.append((d - gt)[mask].abs().cpu().numpy())
    e = np.concatenate(errs)
    return {"covered_px": covered, "median_mm": round(float(np.median(e)) * 1e3, 4),
            "p95_mm": round(float(np.percentile(e, 95)) * 1e3, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--calls", type=int, default=10)
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
    tri, _ = rec.triangulate()
    fill, _ = rec.fill_holes(tri, HoleParams(8, 90.0, 180.0))
    mesh = torch.cat([tri, fill])
    frames = (first + 10, (first + last) // 2, last - 4)
    result = {"card": card(), "surfels_size": rec.surfels_size(), "triangles": len(mesh),
              "triangulate": event_ms(rec.triangulate, args.calls),
              "full_mesh_depth_error": depth_error(rec, cam, st, mesh, frames), "simplify": {}}
    out = torch.empty((len(mesh), 3), dtype=torch.int32, device="cuda")
    configs = {"default max_cost": SimplifyParams.defaults()}
    for pct in (50, 25, 10):
        configs[f"target {pct}%"] = SimplifyParams.defaults(target_triangles=len(mesh) * pct // 100,
                                                            max_cost=float("inf"))
    for name, p in configs.items():
        stats = _lib.SimplifyStats()

        def direct():
            lib.call("mesh_simplify", rec._h, None, C.byref(p), C.c_void_p(mesh.data_ptr()), len(mesh),
                     C.c_void_p(out.data_ptr()), len(out), C.byref(stats))

        direct()
        entry = {k: (float(getattr(stats, k)) if k == "max_cost_applied" else int(getattr(stats, k)))
                 for k, _ in _lib.SimplifyStats._fields_ if k != "reserved"}
        simplified = out[:stats.triangles_out].clone()
        # collapses per round: the difference of calls that stop after r - 1 and r rounds
        per_round, previous = [], 0
        for r in range(1, entry["rounds"] + 1):
            q = SimplifyParams.defaults(target_triangles=p.target_triangles, max_cost=p.max_cost, max_rounds=r)
            _, s = rec.simplify_mesh(mesh, q)
            per_round.append(int(s.collapses) - previous)
            previous = int(s.collapses)
        entry["collapses_per_round"] = per_round
        entry.update(event_ms(direct, args.calls))
        entry["kernel_ms"] = kernel_split(lib, direct)
        entry["depth_error"] = depth_error(rec, cam, st, simplified, frames)
        result["simplify"][name] = entry
        print(name, json.dumps(entry), flush=True)
    rec.close()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text)


if __name__ == "__main__":
    main()
