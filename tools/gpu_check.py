#!/usr/bin/env python
"""Developer parity probe (run on a GPU): product vs. the reference oracle, stage by
stage, with mismatch statistics; also oracle-vs-oracle to show the reference's own
run-to-run envelope. Not a test: tests/ holds the asserted version of these checks."""
import argparse
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402


def u16(h, w):
    return torch.zeros((h, w), dtype=torch.uint16, device="cuda")


def cmp_exact(name, a, b, mask=None):
    a = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    if a.dtype == np.float32:
        a = a.view(np.uint32)
        b = b.view(np.uint32)
    ne = a != b
    if mask is not None:
        ne = ne & mask
    n = int(ne.sum())
    print(f"  {name:34s} mismatches {n:8d} / {ne.size}" + ("" if n == 0 else "   <-- DIFF"))
    return n


def preprocess_stages(lib, cam, pp, raw, others, mats):
    """Runs the five stages separately through `lib`; returns dict of outputs."""
    H, W = cam.height, cam.width
    A, B, A2, B2, A3 = u16(H, W), u16(H, W), u16(H, W), u16(H, W), u16(H, W)
    normals = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
    radius = torch.zeros((H, W), dtype=torch.float32, device="cuda")
    R.BilateralFilteringAndDepthCutoffCUDA(None, pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor, 0,
                                           pp.bilateral_filter_radius_factor, int(pp.depth_scaling * pp.max_depth),
                                           pp.depth_valid_region_radius, raw, A, lib=lib)
    R.OutlierDepthMapFusionCUDA(None, pp.outlier_filtering_depth_tolerance_factor, A, cam.fx, cam.fy, cam.cx, cam.cy,
                                others, mats, B, required_count=pp.outlier_filtering_required_inliers, lib=lib)
    R.ErodeDepthMapCUDA(None, pp.depth_erosion_radius, B, A2, lib=lib)
    R.ComputeNormalsAndDropBadPixelsCUDA(None, pp.observation_angle_threshold_deg, pp.depth_scaling, cam.fx, cam.fy,
                                         cam.cx, cam.cy, A2, B2, normals, lib=lib)
    R.ComputePointRadiiAndRemoveIsolatedPixelsCUDA(None, pp.point_radius_extension_factor,
                                                   pp.point_radius_clamp_factor, pp.depth_scaling, cam.fx, cam.fy,
                                                   cam.cx, cam.cy, B2, radius, A3, lib=lib)
    torch.cuda.synchronize()
    return dict(bilateral=A, outlier=B, erode=A2, normals_depth=B2, normals=normals, radius=radius, final=A3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=28)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--sigma", type=float, default=None)
    ap.add_argument("--cap", type=int, default=2_000_000)
    ap.add_argument("--bench-frames", type=int, default=0)
    args = ap.parse_args()

    prod = _lib.load_product()
    ref = _lib.load_reference_oracle()
    print(prod.version(), "|", ref.version())
    cam = S.Camera.tum(args.width, args.height)
    t0 = time.time()
    st = S.make_stream(cam, args.frames, device="cuda", sigma_depth=args.sigma)
    print(f"stream {args.frames} frames generated in {time.time() - t0:.1f}s")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    K = pp.outlier_filtering_frame_count
    first, last = st.integrated_range()
    H, W = cam.height, cam.width

    # ---- stage-by-stage preprocessing parity ----
    total = 0
    for frame in (first, first + 3):
        print(f"[preprocess stages] frame {frame}")
        others = [st.depth[frame - (i + 1)] for i in range(K // 2)] + [st.depth[frame + (i + 1)] for i in range(K // 2)]
        mats = st.others_TR_reference[frame]
        a = preprocess_stages(ref, cam, pp, st.depth[frame], others, mats)
        # teacher-forced: each product stage consumes the oracle's previous stage
        Hh = lambda: u16(H, W)
        m = {}
        m["bilateral"] = Hh()
        R.BilateralFilteringAndDepthCutoffCUDA(None, pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor,
                                               0, pp.bilateral_filter_radius_factor, int(pp.depth_scaling * pp.max_depth),
                                               pp.depth_valid_region_radius, st.depth[frame], m["bilateral"])
        m["outlier"] = Hh()
        R.OutlierDepthMapFusionCUDA(None, pp.outlier_filtering_depth_tolerance_factor, a["bilateral"], cam.fx, cam.fy,
                                    cam.cx, cam.cy, others, mats, m["outlier"])
        m["erode"] = Hh()
        R.ErodeDepthMapCUDA(None, pp.depth_erosion_radius, a["outlier"], m["erode"])
        m["normals_depth"] = Hh()
        m["normals"] = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
        R.ComputeNormalsAndDropBadPixelsCUDA(None, pp.observation_angle_threshold_deg, pp.depth_scaling, cam.fx, cam.fy,
                                             cam.cx, cam.cy, a["erode"], m["normals_depth"], m["normals"])
        m["final"] = Hh()
        m["radius"] = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        R.ComputePointRadiiAndRemoveIsolatedPixelsCUDA(None, pp.point_radius_extension_factor,
                                                       pp.point_radius_clamp_factor, pp.depth_scaling, cam.fx, cam.fy,
                                                       cam.cx, cam.cy, a["normals_depth"], m["radius"], m["final"])
        torch.cuda.synchronize()
        print("   valid px: raw %d bilateral %d outlier %d erode %d normals %d final %d" % tuple(
            int((x != 0).sum()) for x in (st.depth[frame], a["bilateral"], a["outlier"], a["erode"],
                                          a["normals_depth"], a["final"])))
        for k in ("bilateral", "outlier", "erode", "normals_depth", "normals", "final"):
            total += cmp_exact(k, m[k], a[k])
        rmask = (a["normals_depth"] != 0).cpu().numpy()
        total += cmp_exact("radius (where written)", m["radius"], a["radius"], rmask)

    # ---- fused preprocess vs oracle chain ----
    rec_p = R.CUDASurfelReconstruction(args.cap, W, H, cam.fx, cam.fy, cam.cx, cam.cy)
    rec_a = R.CUDASurfelReconstruction(args.cap, W, H, cam.fx, cam.fy, cam.cx, cam.cy, lib=ref)
    rec_b = R.CUDASurfelReconstruction(args.cap, W, H, cam.fx, cam.fy, cam.cx, cam.cy, lib=ref)

    def run_pre(rec, frame):
        others = [st.depth[frame - (i + 1)] for i in range(K // 2)] + [st.depth[frame + (i + 1)] for i in range(K // 2)]
        d = u16(H, W)
        n = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
        r = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        rec.preprocess(None, pp, st.depth[frame], others, st.others_TR_reference[frame], d, n, r)
        torch.cuda.synchronize()
        return d, n, r

    print("[fused preprocess]")
    for frame in (first, first + 2):
        dp, np_, rp = run_pre(rec_p, frame)
        da, na, ra = run_pre(rec_a, frame)
        total += cmp_exact("depth", dp, da)
        total += cmp_exact("normals", np_, na)
        total += cmp_exact("radius (depth!=0)", rp, ra, (da != 0).cpu().numpy())

    # ---- integrate, teacher forced on oracle A; oracle B = envelope ----
    print("[integrate, teacher-forced]")
    for frame in range(first, last):
        da, na, ra = run_pre(rec_a, frame)
        rows_a, n_a, m_a = rec_a.dump_state()
        rec_p.load_state(rows_a, m_a)
        rec_b.load_state(rows_a, m_a)
        depths = {}
        for name, rec in (("p", rec_p), ("a", rec_a), ("b", rec_b)):
            d = da.clone()
            rec.integrate(None, frame, ip, d, na, ra, st.color[frame], st.global_T_frame[frame], st.frame_T_global[frame])
            torch.cuda.synchronize()
            depths[name] = d
        ras = {k: rec.download_rasters() for k, rec in (("p", rec_p), ("a", rec_a), ("b", rec_b))}
        sts = {k: rec.dump_state() for k, rec in (("p", rec_p), ("a", rec_a), ("b", rec_b))}
        print(f" frame {frame}: N before {n_a}  after p/a/b {sts['p'][1]}/{sts['a'][1]}/{sts['b'][1]}  merges {sts['p'][2]}/{sts['a'][2]}/{sts['b'][2]}")
        for other in ("p", "b"):
            tag = "product" if other == "p" else "oracleB"
            print(f"  -- {tag} vs oracle A")
            for k in ("first_surfel_depth", "supporting_surfel_counts", "conflicting_surfels", "new_surfel_flag_vector",
                      "new_surfel_indices"):
                total += cmp_exact(k, ras[other][k], ras["a"][k]) if other == "p" else cmp_exact(k, ras[other][k], ras["a"][k]) * 0
            sup_o, sup_a, cnt = ras[other]["supporting_surfels"], ras["a"]["supporting_surfels"], ras["a"]["supporting_surfel_counts"]
            cmp_exact("supporting (count==1)", sup_o, sup_a, cnt == 1)
            cmp_exact("supporting (count>1)", sup_o, sup_a, cnt > 1)
            cmp_exact("supporting INV pattern", sup_o == 0xFFFFFFFF, sup_a == 0xFFFFFFFF)
            s_o, s_a = ras[other]["supporting_surfel_depth_sums"], ras["a"]["supporting_surfel_depth_sums"]
            rel = np.abs(s_o - s_a) / np.maximum(np.abs(s_a), 1e-20)
            print(f"  depth sums max rel diff {rel.max():.3e}")
            cmp_exact("blended depth", depths[other], depths["a"])
            ro, ra_ = sts[other][0], sts["a"][0]
            if ro.shape == ra_.shape:
                same_merge = (ro[7] < 0) == (ra_[7] < 0)
                print(f"    surfels with different merge status: {int((~same_merge).sum())}")
                det_rows = (0, 1, 2, 6, 7, 8, 9, 10, 17, 18, 24)
                bad = 0
                for row in det_rows:
                    bad += int(((ro[row].view(np.uint32) != ra_[row].view(np.uint32)) & same_merge).sum())
                print(f"    integrate rows (x,y,z,conf,r2,normal,stamps,color) diffs outside merge differences: {bad}"
                      + ("" if bad == 0 else "   <-- DIFF"))
                if other == "p":
                    total += bad
                for row in (3, 4, 5, 19, 20, 21, 22):
                    ne = (ro[row].view(np.uint32) != ra_[row].view(np.uint32))
                    extra = f" max abs {np.nanmax(np.abs(ro[row] - ra_[row])):.3e}" if row < 6 else ""
                    print(f"    row {row:2d} {R.ROW_NAMES[row]:12s} differs at {int(ne.sum()):6d} (new surfels: {int(ne[n_a:].sum())}){extra}")
            else:
                print("    state shapes differ", ro.shape, ra_.shape)

    # ---- throughput probe ----
    if args.bench_frames > 0:
        print("[throughput probe]")
        stb = S.make_stream(cam, args.bench_frames, device="cuda")
        f0, f1 = stb.integrated_range()
        for name, lib in (("reference", ref), ("product", prod)):
            rec = R.CUDASurfelReconstruction(args.cap, W, H, cam.fx, cam.fy, cam.cx, cam.cy, lib=lib)
            for rep in range(3):
                rec.reset()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                stats = rec.stream_run(None, stb.depth, stb.color, stb.global_T_frame, stb.frame_T_global,
                                       stb.others_TR_reference, pp, ip, f0, f1)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1)
                print(f"  {name:9s} rep {rep}: {stats.frames_integrated} frames {ms:8.2f} ms -> {stats.frames_integrated / ms * 1e3:9.1f} fps;"
                      f" surfels {stats.surfels_size} (count {stats.surfel_count}) launches {stats.kernel_launches}")
            rec.close()
    print("TOTAL hard mismatches:", total)


if __name__ == "__main__":
    main()
