#!/usr/bin/env python
"""sm_render_mesh_textured on the final cloud of the 500-frame VGA synthetic stream (the bench workload), meshed by
sm_triangulate with the holes of up to 8 edges filled, full and simplified with the default sm_mesh_simplify
parameters, each textured at 4 mm from every 10th integrated frame. At VGA and 1920x1080 (the same field of view)
from held-out poses:
  * call time (median and p90 of CUDA events around one synchronised call) of render_mesh and of the textured render,
    alternated in one loop, with the disks of unmeshed surfels; with --parent LIB also render_mesh and
    sm_mesh_texture of another build of the library (the parent commit's) on the same state, alternated with this
    build's;
  * the kernel split of both calls from a separate profiled pass (sm_profile_kernels), hence the resolve's share;
  * the held-out colour error (median and mean of the per-channel absolute error over the triangle pixels) of the
    textured render and of per-vertex colour;
  * a few PNGs (textured, per-vertex, the frame) under --png-dir.
Prints the card name and power limit read in the same run.

    python tools/mesh_render_textured_probe.py [--frames 500] [--calls 50] [--parent variants/lib_parent.so]
        [--out probe_out/mesh_render_textured_probe.json] [--png-dir probe_out/textured_png]
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
from surfelmeshing_b200 import _lib, mesh_io, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import (HoleParams, IntegrateParams, PreprocessParams, SimplifyParams,  # noqa: E402
                                     TextureParams)
from tests.test_mesh_texture_gpu import stream_views  # noqa: E402
from tools.ab_probe import load_build  # noqa: E402
from tools.mesh_update_probe import card  # noqa: E402

CAP = 5_000_000


def event_ms(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def summary(times):
    return {"median_ms": round(float(np.median(times)), 4), "p90_ms": round(float(np.percentile(times, 90)), 4)}


def alternate(fns, calls):
    """Each of fns once to warm up, then `calls` rounds of one call of each, in turn."""
    for fn in fns.values():
        fn()
    times = {k: [] for k in fns}
    for _ in range(calls):
        for k, fn in fns.items():
            times[k].append(event_ms(fn))
    return {k: summary(v) for k, v in times.items()}


def kernel_split(lib, fn):
    lib.fn["profile_kernels"](1)
    fn()
    torch.cuda.synchronize()
    count = lib.fn["profile_kernel_count"]()
    ms, calls = (C.c_double * count)(), (C.c_uint64 * count)()
    lib.fn["profile_report"](ms, calls, count)
    lib.fn["profile_kernels"](0)
    names = [lib.fn["profile_kernel_name"](k).decode() for k in range(count)]
    per = {names[k]: round(ms[k], 4) for k in range(count) if calls[k] and names[k].startswith("k_mesh_render")}
    total = sum(per.values())
    return {"kernels_ms": per, "resolve_share": round(per.get("k_mesh_render_resolve", 0.0) / total, 3) if total else None}


def colour_errors(rec, tri, texture, st, frames, cam):
    tex_err, vert_err = [], []
    for f in frames:
        kw = dict(near=0.1, far=20.0, unmeshed_surfels=False, **cam)
        tex = rec.render_mesh(tri, st.frame_T_global[f], texture=texture, outputs=("color", "index"), **kw)
        vert = rec.render_mesh(tri, st.frame_T_global[f], outputs=("color",), **kw)
        hit = tex["index"] >= 0
        truth = st.color[f].float()
        tex_err.append((tex["color"].float() - truth)[hit].abs().flatten())
        vert_err.append((vert["color"].float() - truth)[hit].abs().flatten())
    tex_err, vert_err = torch.cat(tex_err).cpu().numpy(), torch.cat(vert_err).cpu().numpy()
    return {"median": {"textured": float(np.median(tex_err)), "per_vertex": float(np.median(vert_err))},
            "mean": {"textured": round(float(tex_err.mean()), 3), "per_vertex": round(float(vert_err.mean()), 3)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--texture-calls", type=int, default=5)
    ap.add_argument("--parent", type=Path, default=None, help="another build of the library, timed alternately")
    ap.add_argument("--out", type=Path, default=None)
    ap.add_argument("--png-dir", type=Path, default=None)
    args = ap.parse_args()
    result = {"card": card()}
    lib = _lib.load_product()
    cam = S.Camera.tum(640, 480)
    st = S.make_stream(cam, args.frames, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    rec = R.CUDASurfelReconstruction(CAP, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                   IntegrateParams.defaults(), first, last)
    tri, _ = rec.triangulate()
    full = torch.cat([tri, rec.fill_holes(tri, HoleParams(8, 90.0, 180.0))[0]])
    simple, _ = rec.simplify_mesh(full, SimplifyParams.defaults())
    views = stream_views(st, range(first, last, 10))
    held_out = list(range(first + 5, last, 40))
    p = TextureParams.defaults(texel_size=0.004)
    parent = None
    if args.parent is not None:
        parent_lib = load_build(args.parent)
        parent = R.CUDASurfelReconstruction(CAP, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=parent_lib)
        rows, _, merges = rec.dump_state()
        parent.load_state(rows, merges)
    result.update(surfels_size=rec.surfels_size(), views=len(views), held_out_frames=len(held_out), meshes={})
    vga = dict(width=640, height=480, fx=cam.fx, fy=cam.fy, cx=cam.cx, cy=cam.cy)
    s = 1080 / 480   # 1920 x 1080 with VGA's vertical field of view
    hd = dict(width=1920, height=1080, fx=cam.fx * s, fy=cam.fy * s, cx=960.0, cy=540.0)
    pose = st.frame_T_global[held_out[len(held_out) // 2]]
    for name, mesh in (("full", full), ("simplified", simple)):
        atlas, uv, stats = rec.texture_mesh(mesh, views, p)
        entry = {"triangles": len(mesh), "atlas": [int(stats.atlas_width), int(stats.atlas_height)],
                 "held_out_colour_error": colour_errors(rec, mesh, (atlas, uv), st, held_out, vga)}
        for size, c in (("640x480", vga), ("1920x1080", hd)):
            kw = dict(near=0.1, far=20.0, **c)
            fns = {"render_mesh": lambda: rec.render_mesh(mesh, pose, **kw),
                   "render_mesh_textured": lambda: rec.render_mesh(mesh, pose, texture=(atlas, uv), **kw)}
            if parent is not None:
                fns["render_mesh_parent"] = lambda: parent.render_mesh(mesh, pose, **kw)
            entry[size] = {"call": alternate(fns, args.calls),
                           "split_render_mesh": kernel_split(lib, fns["render_mesh"]),
                           "split_textured": kernel_split(lib, fns["render_mesh_textured"])}
            if parent is not None:
                entry[size]["split_render_mesh_parent"] = kernel_split(parent.lib, fns["render_mesh_parent"])
            print(name, size, json.dumps(entry[size]), flush=True)
        if parent is not None:
            tex_fns = {"texture_mesh": lambda: rec.texture_mesh(mesh, views, p),
                       "texture_mesh_parent": lambda: parent.texture_mesh(mesh, views, p)}
            entry["texture_mesh_call"] = alternate(tex_fns, args.texture_calls)
            print(name, "texture_mesh", json.dumps(entry["texture_mesh_call"]), flush=True)
        if args.png_dir is not None:
            args.png_dir.mkdir(parents=True, exist_ok=True)
            f = held_out[len(held_out) // 2]
            kw = dict(near=0.1, far=20.0, unmeshed_surfels=False, outputs=("color",), **vga)
            tex = rec.render_mesh(mesh, st.frame_T_global[f], texture=(atlas, uv), **kw)["color"]
            vert = rec.render_mesh(mesh, st.frame_T_global[f], **kw)["color"]
            mesh_io.write_png(args.png_dir / f"{name}_textured_f{f}.png", tex.cpu().numpy())
            mesh_io.write_png(args.png_dir / f"{name}_per_vertex_f{f}.png", vert.cpu().numpy())
            mesh_io.write_png(args.png_dir / f"frame_f{f}.png", st.color[f].cpu().numpy())
            hd_tex = rec.render_mesh(mesh, pose, texture=(atlas, uv), **dict(kw, **hd))["color"]
            mesh_io.write_png(args.png_dir / f"{name}_textured_1920x1080.png", hd_tex.cpu().numpy())
        result["meshes"][name] = entry
        del atlas, uv
    rec.close()
    if parent is not None:
        parent.close()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(text)


if __name__ == "__main__":
    main()
