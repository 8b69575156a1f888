#!/usr/bin/env python
"""sm_render_mesh on the final cloud of the 500-frame VGA bench stream (bench.py's stream: stream_id 0, nominal
noise, 5 M surfel cap) and its sm_triangulate mesh, beside sm_render_surfels on the same views.

Views are those of tools/render_probe.py: --poses input poses (evenly spaced integrated frames) and --poses orbit
poses (the input eye turned about the world z axis and raised, looking at the desk), at VGA and at 1280x960. Per
view:
  * us_mesh / us_disks: CUDA events around --reps back-to-back calls (sm_render_mesh with the unmeshed surfels,
    sm_render_surfels) on preallocated outputs after --warmup calls, divided by --reps;
  * the kernel split of sm_render_mesh from a separate profiling pass (sm_profile_kernels: events around every
    launch, so the sum is above the un-profiled time);
  * triangles drawn (passing T1-T3 and covering a pixel centre) and unmeshed disks drawn, from the plain-C
    restatement (tests/mesh_render_walk.c), and triangles listed as large (a float32 numpy restatement of the
    rectangle rule of render.cu);
  * median and 95th percentile of |render - ground truth| depth where both have depth, and the share of
    ground-truth pixels covered, for the mesh and for the disks (ground truth: the float64 ray cast of the scene).
Writes PNGs (mesh colour, triangle-normal shading, depth error 0-2 cm) of the first --images poses of each kind and
size to --out, and one JSON summary with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from render_probe import card, write_png  # noqa: E402
from surfelmeshing_b200 import synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, RENDER_UNMESHED_SURFELS, RenderParams  # noqa: E402
from tests import mesh_render_walk as MRW  # noqa: E402

NEAR, FAR = 0.1, 20.0
SMALL_TRIANGLE_PIXELS = 64   # render.cu kSmallTrianglePixels
KERNELS = ("k_mesh_render_mark", "k_mesh_render_tri", "k_mesh_render_large", "k_mesh_render_splat",
           "k_mesh_render_splat_large", "k_mesh_render_resolve")


def large_triangles(rows, n, tris, T, c):
    """Triangles whose screen rectangle (render.cu triangle_rect) has more than SMALL_TRIANGLE_PIXELS pixels."""
    t = tris.astype(np.int64)
    present = (t < n).all(1)
    t = t[present]
    present = (rows[7][t] > 0).all(1)
    t = t[present]
    p = rows[3:6].T.astype(np.float32)
    Tm = np.asarray(T, np.float32).reshape(3, 4)
    cam = (p @ Tm[:, :3].T + Tm[:, 3]).astype(np.float32)
    z = cam[:, 2]
    u = (np.float32(c.fx) * (cam[:, 0] / z) + np.float32(c.cx)).astype(np.float32)
    v = (np.float32(c.fy) * (cam[:, 1] / z) + np.float32(c.cy)).astype(np.float32)
    ok = ((z[t] >= NEAR) & (z[t] <= FAR)).all(1)
    t = t[ok]

    def axis(lo, hi, size):
        pad = 1.0 + (np.abs(lo) + np.abs(hi)) * 1e-6
        q0 = np.maximum(np.floor(lo - 0.5 - pad), 0)
        q1 = np.minimum(np.ceil(hi - 0.5 + pad), size - 1)
        return np.where(q0 <= q1, q1 - q0 + 1, 0)

    with np.errstate(invalid="ignore", over="ignore"):
        w = axis(u[t].min(1), u[t].max(1), c.width)
        h = axis(v[t].min(1), v[t].max(1), c.height)
    return int((w * h > SMALL_TRIANGLE_PIXELS).sum())


def depth_error(depth, gt):
    gt_valid = torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0)
    both = gt_valid & (depth > 0)
    err = (depth - gt)[both].abs().cpu().numpy()
    return (float(np.median(err)) if err.size else None, float(np.percentile(err, 95)) if err.size else None,
            float(both.sum()) / max(float(gt_valid.sum()), 1.0), both)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--cap", type=int, default=5_000_000)
    ap.add_argument("--poses", type=int, default=20)
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--images", type=int, default=2, help="poses of each kind and size written as PNG")
    ap.add_argument("--out", default="probe_out/mesh_render")
    args = ap.parse_args()
    out_dir = Path(args.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    cam = S.Camera.tum(640, 480)
    st = S.make_stream(cam, args.frames, stream_id=0, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    rec = R.CUDASurfelReconstruction(args.cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    first, last = st.integrated_range()
    rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                   first, last)
    rows, n, _ = rec.dump_state()
    rows = rows.copy()
    tris, mstats = rec.triangulate()
    tris_host = tris.cpu().numpy()
    print(f"{n} slots, {tris.shape[0]} triangles, {mstats.vertices_meshed} slots meshed", flush=True)
    poses64 = S.trajectory(args.frames)
    frames = np.linspace(first, last - 1, args.poses).round().astype(int)
    views = [("input", int(f), poses64[f]) for f in frames]
    for k, f in enumerate(frames):
        eye = poses64[f][:, 3]
        a = np.radians(25.0 + 10.0 * (k % 4))
        rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        views.append(("orbit", int(f), S._look_at(rz @ eye + np.array([0.0, 0.0, 0.3]), np.array([0.0, 0.0, 0.8]))))
    cams = {"640x480": cam, "1280x960": S.Camera.tum(1280, 960)}
    lib = rec.lib
    nk = lib.fn["profile_kernel_count"]()
    names = [lib.fn["profile_kernel_name"](i).decode() for i in range(nk)]
    kid = {nm: i for i, nm in enumerate(names)}
    handle = torch.cuda.current_stream().cuda_stream
    results, written = [], {}
    for size, c in cams.items():
        camkw = dict(width=c.width, height=c.height, fx=c.fx, fy=c.fy, cx=c.cx, cy=c.cy)
        params = RenderParams(c.width, c.height, c.fx, c.fy, c.cx, c.cy, NEAR, FAR)
        for kind, f, g64 in views:
            T = R.invert_rigid(g64)
            Tc = np.ascontiguousarray(T.reshape(-1)[:12])
            mesh = rec.render_mesh(tris, T, near=NEAR, far=FAR, **camkw)
            disks = rec.render(T, near=NEAR, far=FAR, **camkw)
            raw_m, raw_d = [], []
            for k in R.RENDER_OUTPUTS:
                raw_m += [C.c_void_p(mesh[k].data_ptr()), mesh[k].stride(0) * mesh[k].element_size()]
                raw_d += [C.c_void_p(disks[k].data_ptr()), disks[k].stride(0) * disks[k].element_size()]

            def call_mesh():
                lib.fn["render_mesh"](rec._h, handle, C.byref(params), Tc.ctypes.data_as(C.c_void_p),
                                      C.c_void_p(tris.data_ptr()), tris.shape[0], RENDER_UNMESHED_SURFELS, *raw_m)

            def call_disks():
                lib.fn["render_surfels"](rec._h, handle, C.byref(params), Tc.ctypes.data_as(C.c_void_p), *raw_d)

            times = {}
            for name, fn in (("us_mesh", call_mesh), ("us_disks", call_disks)):
                for _ in range(args.warmup):
                    fn()
                start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                start.record()
                for _ in range(args.reps):
                    fn()
                stop.record()
                torch.cuda.synchronize()
                times[name] = start.elapsed_time(stop) * 1e3 / args.reps
            lib.call("profile_kernels", 1)
            for _ in range(10):
                call_mesh()
            torch.cuda.synchronize()
            tot = np.zeros(nk, np.float64)
            cnt = np.zeros(nk, np.uint64)
            lib.call("profile_report", tot.ctypes.data_as(C.POINTER(C.c_double)),
                     cnt.ctypes.data_as(C.POINTER(C.c_uint64)), nk)
            lib.call("profile_kernels", 0)
            split = {nm: float(tot[kid[nm]] / max(int(cnt[kid[nm]]), 1) * 1e3) for nm in KERNELS}
            _, counts = MRW.render(rows, tris_host, T, c.width, c.height, c.fx, c.fy, c.cx, c.cy, NEAR, FAR,
                                   unmeshed_surfels=True, stats=True)
            gt, _ = S._raycast(c, torch.from_numpy(g64).to("cuda"), "cuda")
            m_med, m_p95, m_cov, both = depth_error(mesh["depth"].double(), gt)
            d_med, d_p95, d_cov, _ = depth_error(disks["depth"].double(), gt)
            tri_px = int(((mesh["index"] >= 0) & (mesh["depth"] > 0)).sum())
            r = {"size": size, "kind": kind, "frame": f, **times, "split_us_profiled": split,
                 "triangles_drawn": counts["triangles"], "triangles_large": large_triangles(rows, n, tris_host, T, c),
                 "disks_drawn": counts["disks"], "pixels_by_triangles": tri_px,
                 "mesh_err_median_m": m_med, "mesh_err_p95_m": m_p95, "mesh_gt_coverage": m_cov,
                 "disk_err_median_m": d_med, "disk_err_p95_m": d_p95, "disk_gt_coverage": d_cov}
            results.append(r)
            print(json.dumps(r), flush=True)
            key = (size, kind)
            if written.get(key, 0) < args.images:
                written[key] = written.get(key, 0) + 1
                stem = out_dir / f"{size}_{kind}_f{f:03d}"
                write_png(f"{stem}_color.png", mesh["color"].cpu().numpy())
                write_png(f"{stem}_shaded.png", R.shade_normals(mesh["normal"]).cpu().numpy())
                e = torch.where(both, (mesh["depth"].double() - gt).abs(), torch.zeros_like(gt)).cpu().numpy()
                write_png(f"{stem}_depth_error.png", (e / 0.02 * 255.0).clip(0, 255))
    summary = {"card": card(), "surfels_size": n, "triangles": int(tris.shape[0]), "frames": args.frames,
               "reps": args.reps, "renders": {}}
    for size in cams:
        for kind in ("input", "orbit"):
            sel = [r for r in results if r["size"] == size and r["kind"] == kind]
            med = lambda key: float(np.median([r[key] for r in sel]))  # noqa: E731
            summary["renders"][f"{size} {kind}"] = {
                "us_mesh_median": med("us_mesh"), "us_mesh_p90": float(np.percentile([r["us_mesh"] for r in sel], 90)),
                "us_disks_median": med("us_disks"),
                "us_disks_p90": float(np.percentile([r["us_disks"] for r in sel], 90)),
                "split_us_median": {k: float(np.median([r["split_us_profiled"][k] for r in sel])) for k in KERNELS},
                "triangles_drawn_median": med("triangles_drawn"), "triangles_large_median": med("triangles_large"),
                "disks_drawn_median": med("disks_drawn"),
                "mesh_err_median_m": med("mesh_err_median_m"), "mesh_err_p95_m": med("mesh_err_p95_m"),
                "mesh_gt_coverage": med("mesh_gt_coverage"),
                "disk_err_median_m": med("disk_err_median_m"), "disk_err_p95_m": med("disk_err_p95_m"),
                "disk_gt_coverage": med("disk_gt_coverage")}
    print(json.dumps(summary, indent=1))
    (out_dir / "summary.json").write_text(json.dumps({"summary": summary, "renders": results}, indent=1))


if __name__ == "__main__":
    main()
