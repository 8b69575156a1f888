#!/usr/bin/env python
"""sm_render_surfels on the final cloud of the 500-frame VGA bench stream (bench.py's stream: stream_id 0, nominal
noise, 5 M surfel cap).

The stream is integrated with sm_stream_run, then the cloud is rendered from --poses input poses (evenly spaced
integrated frames) and --poses off-trajectory poses (the input eye turned about the world z axis and raised, looking
at the desk), at VGA and at 1280x960 (the same camera scaled). Per render:
  * us: CUDA events around --reps back-to-back renders after --warmup renders, divided by --reps;
  * the split between k_render_splat, k_render_large and k_render_resolve, from a separate profiling pass
    (sm_profile_kernels: events around every launch, so the sum is above the un-profiled time);
  * surfels drawn, pixels tested and large splats, counted on the host from the dumped state with the kernels'
    rectangle rule (a float32 numpy restatement of render.cu's load_splat);
  * algorithmic bytes: 32 B per slot for the sweep (one 16-byte record and rows 7-10), and per pixel the 8-byte
    key, the 23 output bytes and, for covered pixels, the key reset and the winner's 16 bytes of colour and normal;
    over the measured time;
  * median and 95th percentile of |render - ground truth| depth where both have depth, and the share of
    ground-truth pixels covered (ground truth: the float64 ray cast of the scene, synthetic._raycast).
Writes PNGs of colour, depth (normalised to [near, far] of the image), normals and the depth error (0-2 cm) of the
first two poses of each kind and size to --out, and one JSON summary with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import struct
import subprocess
import sys
import zlib
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams, RenderParams  # noqa: E402

NEAR, FAR = 0.1, 20.0
SMALL_SPLAT_PIXELS = 64   # render.cu kSmallSplatPixels


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[torch.cuda.current_device()] if out.returncode == 0 else "unknown"


def write_png(path, img):
    """8-bit grey [H, W] or RGB [H, W, 3] PNG with zlib and struct only."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape[:2]
    colour_type = 2 if img.ndim == 3 else 0
    raw = b"".join(b"\x00" + img[y].tobytes() for y in range(h))

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    Path(path).write_bytes(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, colour_type, 0, 0, 0)) +
                           chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def splat_counts(rows, T, cam):
    """(surfels drawn, pixels tested, large splats) with render.cu's rectangle rule, in float32."""
    f32 = np.float32
    T = np.asarray(T, f32).reshape(3, 4)
    r2 = rows[7]
    s = rows[3:6]
    c = [(s[1] * T[k, 1] + s[0] * T[k, 0] + s[2] * T[k, 2] + T[k, 3]).astype(f32) for k in range(3)]
    drawn = (r2 > 0) & (c[2] >= f32(NEAR)) & (c[2] <= f32(FAR))
    r2, c = r2[drawn], [v[drawn] for v in c]
    reach = (np.sqrt(r2) * f32(1.0001) + (np.abs(c[0]) + np.abs(c[1]) + np.abs(c[2])) * f32(1e-5)).astype(f32)
    z_lo, z_hi = c[2] - reach, c[2] + reach
    whole = ~(z_lo > 0)
    zl = np.where(whole, f32(1), z_lo)

    def axis(cc, f, pc, size):
        lo, hi = cc - reach, cc + reach
        d_min = np.where(lo >= 0, lo / z_hi, lo / zl)
        d_max = np.where(hi >= 0, hi / zl, hi / z_hi)
        q0 = np.floor(f * d_min + (pc - f32(0.5))) - 1
        q1 = np.ceil(f * d_max + (pc - f32(0.5))) + 1
        q0, q1 = np.maximum(q0, 0), np.minimum(q1, size - 1)
        return np.where(whole, 0, q0), np.where(whole, size - 1, q1)

    x0, x1 = axis(c[0], f32(cam.fx), f32(cam.cx), cam.width)
    y0, y1 = axis(c[1], f32(cam.fy), f32(cam.cy), cam.height)
    inside = (x0 <= x1) & (y0 <= y1)
    pixels = ((x1 - x0 + 1) * (y1 - y0 + 1)).astype(np.int64)[inside]
    return int(inside.sum()), int(pixels.sum()), int((pixels > SMALL_SPLAT_PIXELS).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--cap", type=int, default=5_000_000)
    ap.add_argument("--poses", type=int, default=20)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--images", type=int, default=2, help="poses of each kind and size written as PNG")
    ap.add_argument("--out", default="probe_out/render")
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
    poses64 = S.trajectory(args.frames)
    frames = np.linspace(first, last - 1, args.poses).round().astype(int)
    views = []   # (kind, frame, camera-to-world float64)
    for f in frames:
        views.append(("input", int(f), poses64[f]))
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
    results = []
    written = {}
    for size, c in cams.items():
        camkw = dict(width=c.width, height=c.height, fx=c.fx, fy=c.fy, cx=c.cx, cy=c.cy)
        P = c.width * c.height
        for kind, f, g64 in views:
            T = R.invert_rigid(g64)
            for _ in range(args.warmup):
                rec.render(T, near=NEAR, far=FAR, **camkw)
            bufs = rec.render(T, near=NEAR, far=FAR, **camkw)
            # the timed loop calls the C ABI on preallocated outputs (no allocation between launches)
            params = RenderParams(c.width, c.height, c.fx, c.fy, c.cx, c.cy, NEAR, FAR)
            Tc = np.ascontiguousarray(T.reshape(-1)[:12])
            raw = []
            for k in R.RENDER_OUTPUTS:
                raw += [C.c_void_p(bufs[k].data_ptr()), bufs[k].stride(0) * bufs[k].element_size()]
            handle = torch.cuda.current_stream().cuda_stream
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            for _ in range(args.reps):
                lib.fn["render_surfels"](rec._h, handle, C.byref(params), Tc.ctypes.data_as(C.c_void_p), *raw)
            stop.record()
            torch.cuda.synchronize()
            us = start.elapsed_time(stop) * 1e3 / args.reps
            lib.call("profile_kernels", 1)
            for _ in range(20):
                rec.render(T, near=NEAR, far=FAR, **camkw)
            tot = np.zeros(nk, np.float64)
            cnt = np.zeros(nk, np.uint64)
            lib.call("profile_report", tot.ctypes.data_as(C.POINTER(C.c_double)),
                     cnt.ctypes.data_as(C.POINTER(C.c_uint64)), nk)
            lib.call("profile_kernels", 0)
            split = {nm: float(tot[kid[nm]] / max(int(cnt[kid[nm]]), 1) * 1e3)
                     for nm in ("k_render_splat", "k_render_large", "k_render_resolve")}
            drawn, tested, large = splat_counts(rows, T, c)
            depth = bufs["depth"].double()
            covered = int((depth > 0).sum())
            nbytes = 32 * n + P * (8 + 23) + covered * (8 + 16)
            gt, _ = S._raycast(c, torch.from_numpy(g64).to("cuda"), "cuda")
            gt_valid = torch.isfinite(gt) & (gt > 0.3) & (gt < 13.0)
            both = gt_valid & (depth > 0)
            err = (depth - gt)[both].abs().cpu().numpy()
            rec_ = {"size": size, "kind": kind, "frame": f, "us": us, "split_us_profiled": split, "surfels": n,
                    "drawn": drawn, "pixels_tested": tested, "large_splats": large, "covered_pixels": covered,
                    "bytes": nbytes, "GB_per_s": nbytes / (us * 1e-6) / 1e9,
                    "err_median_m": float(np.median(err)) if err.size else None,
                    "err_p95_m": float(np.percentile(err, 95)) if err.size else None,
                    "gt_coverage": float(both.sum()) / max(float(gt_valid.sum()), 1.0)}
            results.append(rec_)
            print(json.dumps(rec_), flush=True)
            key = (size, kind)
            if written.get(key, 0) < args.images:
                written[key] = written.get(key, 0) + 1
                stem = out_dir / f"{size}_{kind}_f{f:03d}"
                write_png(f"{stem}_color.png", bufs["color"].cpu().numpy())
                d = depth.cpu().numpy()
                valid = d > 0
                lo, hi = (d[valid].min(), d[valid].max()) if valid.any() else (0.0, 1.0)
                grey = np.where(valid, 255.0 * (1.0 - (d - lo) / max(hi - lo, 1e-9)), 0.0)
                write_png(f"{stem}_depth.png", grey.clip(0, 255))
                nrm = bufs["normal"].cpu().numpy()
                write_png(f"{stem}_normal.png", np.where(valid[..., None], (nrm + 1.0) * 127.5, 0).clip(0, 255))
                e = torch.where(both, (depth - gt).abs(), torch.zeros_like(depth)).cpu().numpy()
                write_png(f"{stem}_depth_error.png", (e / 0.02 * 255.0).clip(0, 255))
    summary = {"card": card(), "surfels_size": n, "frames": args.frames, "reps": args.reps, "renders": {}}
    for size in cams:
        for kind in ("input", "orbit"):
            sel = [r for r in results if r["size"] == size and r["kind"] == kind]
            us = [r["us"] for r in sel]
            summary["renders"][f"{size} {kind}"] = {
                "us_median": float(np.median(us)), "us_min": float(min(us)), "us_max": float(max(us)),
                "split_us_median": {k: float(np.median([r["split_us_profiled"][k] for r in sel]))
                                    for k in sel[0]["split_us_profiled"]},
                "drawn_median": int(np.median([r["drawn"] for r in sel])),
                "pixels_tested_median": int(np.median([r["pixels_tested"] for r in sel])),
                "large_splats_median": int(np.median([r["large_splats"] for r in sel])),
                "GB_per_s_median": float(np.median([r["GB_per_s"] for r in sel])),
                "err_median_m_median": float(np.median([r["err_median_m"] for r in sel])),
                "err_p95_m_median": float(np.median([r["err_p95_m"] for r in sel])),
                "gt_coverage_median": float(np.median([r["gt_coverage"] for r in sel]))}
    print(json.dumps(summary))
    (out_dir / "summary.json").write_text(json.dumps({"summary": summary, "renders": results}, indent=1))


if __name__ == "__main__":
    main()
