"""sm_mesh_texture on the final cloud of the 500-frame VGA synthetic stream (the bench workload), meshed by
sm_triangulate with the holes of up to 8 edges filled, then simplified with the default sm_mesh_simplify parameters,
textured from every 10th integrated frame: the atlas size and texels at several texel sizes; the time of one call
(median and p90 over synchronised calls, CUDA events around the call, after a warm-up call); the split into layout,
per-view render, accumulation and resolve from a separate profiled call; the scratch it needs, from the sizes;
and the median colour error on held-out frames (textured against per-vertex colour) on the full and the simplified
mesh. Prints the card name and power limit read in the same run.

    python tools/mesh_texture_probe.py [--frames 500] [--calls 10] [--out probe_out/mesh_texture_probe.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import (HoleParams, IntegrateParams, PreprocessParams, SimplifyParams,  # noqa: E402
                                     TextureParams, TextureStats, TextureViewDesc)
from tests.test_mesh_texture_gpu import colour_errors, stream_views  # noqa: E402
from tools.mesh_holes_probe import event_ms  # noqa: E402
from tools.mesh_update_probe import card  # noqa: E402

SPLIT = {"layout": ("k_tex_classes", "k_tex_sort", "k_tex_place", "k_tex_uv"), "accumulate": ("k_tex_accumulate",),
         "resolve": ("k_tex_resolve",)}


def kernel_split(lib, fn):
    lib.fn["profile_kernels"](1)
    fn()
    torch.cuda.synchronize()
    count = lib.fn["profile_kernel_count"]()
    ms, calls = (C.c_double * count)(), (C.c_uint64 * count)()
    lib.fn["profile_report"](ms, calls, count)
    lib.fn["profile_kernels"](0)
    names = [lib.fn["profile_kernel_name"](k).decode() for k in range(count)]
    per = {names[k]: [round(ms[k], 4), int(calls[k])] for k in range(count)
           if calls[k] and names[k].startswith(("k_tex", "k_mesh_render"))}
    split = {part: round(sum(per[k][0] for k in ks if k in per), 4) for part, ks in SPLIT.items()}
    split["render"] = round(sum(v[0] for k, v in per.items() if k.startswith("k_mesh_render")), 4)
    return per, split


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
    view_frames = list(range(first, last, 10))
    held_out = list(range(first + 5, last, 40))
    views = stream_views(st, view_frames)
    descs = (TextureViewDesc * len(views))(*[v.desc() for v in views])
    result = {"card": card(), "surfels_size": rec.surfels_size(), "triangles_full": len(full),
              "triangles_simplified": len(simple), "views": len(views), "held_out_frames": len(held_out),
              "texel_sizes": {}}
    for texel in (0.002, 0.004, 0.008):
        p = TextureParams.defaults(texel_size=texel)
        entry = {}
        for name, mesh in (("simplified", simple), ("full", full)):
            try:
                atlas, uv, stats = rec.texture_mesh(mesh, views, p)
            except _lib.SurfelError as e:
                entry[name] = {"error": str(e)}
                continue
            s = {k: int(getattr(stats, k)) for k, _ in TextureStats._fields_}
            out_stats = TextureStats()

            def direct():
                lib.call("mesh_texture", rec._h, None, C.byref(p), C.c_void_p(mesh.data_ptr()), len(mesh), descs,
                         len(views), C.c_void_p(atlas.data_ptr()), atlas.stride(0), atlas.shape[1], atlas.shape[0],
                         C.c_void_p(uv.data_ptr()), C.byref(out_stats))

            s["call"] = event_ms(direct, args.calls)
            s["kernel_ms"], s["split_ms"] = kernel_split(lib, direct)
            # the call's own scratch, from the sizes (include/surfel_b200.h): accumulators <= 16 B per atlas texel,
            # 24 B per triangle, 4 B per view pixel
            s["scratch_bytes_at_most"] = 16 * stats.atlas_width * stats.atlas_height + 24 * len(mesh) + 4 * 640 * 480
            tex, vert, tex_mean, vert_mean = colour_errors(rec, st, mesh, atlas, uv, held_out)
            s["held_out_median_abs_error"] = {"textured": round(tex, 3), "per_vertex": round(vert, 3)}
            s["held_out_mean_abs_error"] = {"textured": round(tex_mean, 3), "per_vertex": round(vert_mean, 3)}
            entry[name] = s
            print(texel, name, json.dumps(s), flush=True)
            del atlas, uv
        result["texel_sizes"][str(texel)] = entry
    rec.close()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text)


if __name__ == "__main__":
    main()
