"""sm_mesh_texture_compensated on the final cloud of the 500-frame VGA synthetic stream (the bench workload), meshed by
sm_triangulate with the holes of up to 8 edges filled, full and simplified with the default sm_mesh_simplify
parameters, textured at 4 mm texels from every 10th integrated frame (50 views) whose images carry a seeded
simulated auto-exposure and white balance (per view and channel gains in about [0.7, 1.3]). Reports, per mesh:
the time of one call next to sm_mesh_texture's on the same views (median and p90 over synchronised calls, CUDA
events, after a warm-up); the split into sampling renders, sampling, the conjugate-gradient solve, accumulation
renders, accumulation and resolve from separate profiled calls; the gain fit's memory, from the sizes; the gain
error max_v |g_v k_v / median - 1| against the true gains; and the held-out colour error (mean |c x - y| after one
least-squares scale c per channel) with and without compensation. Prints the card name and power limit read in the
same run.

    python tools/mesh_texture_gains_probe.py [--frames 500] [--calls 10] [--out probe_out/mesh_texture_gains.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import (HoleParams, IntegrateParams, PreprocessParams, SimplifyParams,  # noqa: E402
                                     TextureGainParams, TextureGainStats, TextureParams, TextureStats,
                                     TextureViewDesc)
from tests.test_mesh_texture_gains_gpu import held_out_samples, random_walk_gains, scaled_error  # noqa: E402
from tools.mesh_holes_probe import event_ms  # noqa: E402
from tools.mesh_update_probe import card  # noqa: E402

GAIN_KERNELS = ("k_tex_gain_count", "k_tex_gain_points", "k_tex_gain_views", "k_tex_gain_step")


def profile(lib, fn):
    """Per-kernel time (ms) and launches of one call of fn."""
    lib.fn["profile_kernels"](1)
    fn()
    torch.cuda.synchronize()
    count = lib.fn["profile_kernel_count"]()
    ms, calls = (C.c_double * count)(), (C.c_uint64 * count)()
    lib.fn["profile_report"](ms, calls, count)
    lib.fn["profile_kernels"](0)
    names = [lib.fn["profile_kernel_name"](k).decode() for k in range(count)]
    return {names[k]: [round(ms[k], 4), int(calls[k])] for k in range(count)
            if calls[k] and names[k].startswith(("k_tex", "k_mesh_render"))}


def render_ms(per):
    return sum(v[0] for k, v in per.items() if k.startswith("k_mesh_render"))


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
    full = torch.cat([tri, rec.fill_holes(tri, HoleParams(8, 90.0, 180.0))[0]])
    simple, _ = rec.simplify_mesh(full, SimplifyParams.defaults())
    frames = list(range(first, last, 10))
    held_out = list(range(first + 5, last, 40))
    k = random_walk_gains(len(frames), seed=11)
    gained = []
    for v, f in enumerate(frames):
        img = torch.round(st.color[f].to(torch.float64) * torch.as_tensor(k[v], device="cuda")).clamp(0, 255)
        gained.append(img.to(torch.uint8).contiguous())
    views = [R.TextureView(gained[v], cam, view_T_global=st.frame_T_global[f], near=0.1, far=20.0)
             for v, f in enumerate(frames)]
    descs = (TextureViewDesc * len(views))(*[v.desc() for v in views])
    p, gp = TextureParams.defaults(), TextureGainParams.defaults()
    V = len(views)
    result = {"card": card(), "surfels_size": rec.surfels_size(), "triangles_full": len(full),
              "triangles_simplified": len(simple), "views": V, "held_out_frames": len(held_out),
              "gain_params": {f: getattr(gp, f) for f, _ in TextureGainParams._fields_}, "meshes": {}}
    for name, mesh in (("simplified", simple), ("full", full)):
        atlas, uv, stats, gains, gstats = rec.texture_mesh(mesh, views, p, gains=gp)
        plain_atlas, plain_uv, _ = rec.texture_mesh(mesh, views, p)
        out_stats, out_gstats = TextureStats(), TextureGainStats()

        def plain():
            lib.call("mesh_texture", rec._h, None, C.byref(p), C.c_void_p(mesh.data_ptr()), len(mesh), descs, V,
                     C.c_void_p(atlas.data_ptr()), atlas.stride(0), atlas.shape[1], atlas.shape[0],
                     C.c_void_p(uv.data_ptr()), C.byref(out_stats))

        def compensated():
            lib.call("mesh_texture_compensated", rec._h, None, C.byref(p), C.byref(gp), C.c_void_p(mesh.data_ptr()),
                     len(mesh), descs, V, C.c_void_p(atlas.data_ptr()), atlas.stride(0), atlas.shape[1],
                     atlas.shape[0], C.c_void_p(uv.data_ptr()), None, C.byref(out_stats), C.byref(out_gstats))

        s = {"atlas": [stats.atlas_width, stats.atlas_height],
             "gain_stats": {f: getattr(gstats, f) for f, _ in TextureGainStats._fields_}}
        s["call_ms"] = {"sm_mesh_texture": event_ms(plain, args.calls),
                        "sm_mesh_texture_compensated": event_ms(compensated, args.calls)}
        per_plain, per_comp = profile(lib, plain), profile(lib, compensated)
        s["kernel_ms"] = per_comp
        s["split_ms"] = {
            "sampling_renders": round(render_ms(per_comp) - render_ms(per_plain), 4),
            "sampling": per_comp.get("k_tex_gain_sample", [0.0])[0],
            "cg_and_data_terms": round(sum(per_comp[kk][0] for kk in GAIN_KERNELS if kk in per_comp), 4),
            "accumulation_renders": round(render_ms(per_plain), 4),
            "accumulation": per_comp.get("k_tex_accumulate", [0.0])[0],
            "resolve": per_comp.get("k_tex_resolve", [0.0])[0]}
        P = int(gstats.points)
        blocks = math.ceil(P / 1024)
        s["gain_scratch_bytes"] = {"samples": 12 * P * V, "per_point": 28 * P, "column_sums": 24 * V * blocks,
                                   "state": (12 + 4 + 72) * 1024 + 16 + 36}
        # one CG iteration reads the sample matrix twice (the point and the view sweeps)
        s["bytes_per_iteration_sample_matrix"] = 2 * 12 * P * V
        g = gains.numpy().astype(np.float64)
        prod = g * k
        s["gain_error"] = {"compensated": float(np.max(np.abs(prod / np.median(prod, 0) - 1))),
                           "uncompensated": float(np.max(np.abs(k / np.median(k, 0) - 1)))}
        tex_c, truth = held_out_samples(rec, st, mesh, atlas, uv, held_out)
        tex_p, _ = held_out_samples(rec, st, mesh, plain_atlas, plain_uv, held_out)
        s["held_out_scaled_mean_abs_error"] = {"compensated": round(scaled_error(tex_c, truth), 3),
                                               "uncompensated": round(scaled_error(tex_p, truth), 3)}
        result["meshes"][name] = s
        print(name, json.dumps(s), flush=True)
        del atlas, uv, plain_atlas, plain_uv
    result["true_gains"] = k.tolist()
    rec.close()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text)


if __name__ == "__main__":
    main()
