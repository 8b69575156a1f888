#!/usr/bin/env python
"""bench.py — RGB-D frames/s of the per-frame surfel reconstruction hot path on H100.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl product|reference] [--dump-outputs DIR]
  torchrun --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

One STEP = one pass over a whole synthetic TUM-fr1/desk-shaped 640x480 RGB-D stream
(BASELINE.json configs[1]: 500 frames -> 492 integrated frames, 5 M surfel cap): depth
pre-processing (a1-a5) + CUDASurfelReconstruction::Integrate() (a6-a14) per frame, through
the C ABI (sm_stream_run). The surfel cloud is reset before every step, so all steps do the
same work. At N > 1 every rank processes its own stream (BASELINE.json configs[3]: independent
streams, one per GPU, weak scaling, no collective on the data path).

  value : whole-job frames/s with the stream resident in HBM (770 MB of frames per step,
          larger than the 50 MB L2, so no L2 flush is needed between steps)
  e2e   : the same through HOST (pinned) frame buffers: every raw depth map and colour image
          is uploaded inside the timed region (copy stream overlapped with compute, as the
          reference's main loop does) and the CUDASurfelBuffersCPU arrays are transferred back
          at the end of the step (TransferAllToCPU)
  roofline : the dominant kernel of a profiled extra pass (per-kernel CUDA events recorded by
          the library on its launching stream), algorithmic bytes from DESIGN.md §5
  cpu_baseline : oracle/cpu_walk.c (plain C + OpenMP port of the filter chain and of the
          min-depth/association loop; the reference ships no CPU implementation) on a bounded
          sample of the same stream, on the box's host cores

--impl reference runs the reference's OWN kernels (unmodified .cu files rebuilt for sm_90a,
oracle/_ref/libsurfel_ref.so) through the same stream runner and prints the same line with
"impl": "reference". The reference implements this path only in CUDA, so its arm runs on the
same GPU; see DESIGN.md §7.

--dump-outputs DIR writes, after the timed steps, what the last timed step computed: the
CUDASurfelBuffersCPU arrays of the final cloud (TransferAllToCPU), sampled at the surfels nearest
to 262 144 fixed points on the scene's surfaces (slot order is not reproducible, see dump_outputs),
and the step's counts, as DIR/<name>.npy (float32 / float64, fixed shapes). The input stream is
seeded, so two builds can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import os

# The cpu_baseline leg (oracle/cpu_walk.c, OpenMP) is timed on pinned threads: set before the OpenMP
# runtime is loaded.
os.environ.setdefault("OMP_PROC_BIND", "close")
os.environ.setdefault("OMP_PLACES", "cores")
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import distributed as D  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402

METRIC = "RGB-D frames/s at 640x480 (depth pre-processing + Integrate())"


def measured_peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        j = json.loads(p.read_text())
        return float(j["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "H100 SXM data sheet (HBM3, 700 W card)"


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons during the timed region."""

    def __init__(self, gpu_index: int):
        self.gpu = gpu_index
        self.samples = []
        self.reasons = set()
        self._stop = threading.Event()
        self._thread = None

    def _run(self):
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                                      str(self.gpu)], capture_output=True, text=True, timeout=5).stdout.strip()
                f = [x.strip() for x in out.split(",")]
                self.samples.append((float(f[0]), float(f[1])))
                for n, v in zip(names, f[2:]):
                    if v.lower().startswith("active"):
                        self.reasons.add(n)
            except Exception:
                pass
            self._stop.wait(0.2)

    def __enter__(self):
        if os.environ.get("SM_BENCH_NO_CLOCKS") == "1":   # diagnosis only: a line without clocks is not a bench value
            return self
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=6)

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": sorted(self.reasons)}
        sm = sorted(s[0] for s in self.samples)
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": max(s[1] for s in self.samples),
                "reasons": sorted(self.reasons)}


def timed_steps(info, device, step_fn, warmup, steps):
    """W untimed + K timed steps bracketed by barrier + synchronize; device time by CUDA events."""
    for _ in range(warmup):
        step_fn()
    torch.cuda.synchronize(device)
    D.barrier(info, device)
    torch.cuda.synchronize(device)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    last = None
    for _ in range(steps):
        last = step_fn()
    e1.record()
    torch.cuda.synchronize(device)
    D.barrier(info, device)
    return e0.elapsed_time(e1), last


def algorithmic_bytes(kernel, c):
    """DESIGN.md §5: algorithmic bytes of one launch. c: P, K, valid, N, V, S, M, A."""
    P, K, N, V, S_, M, A, D = c["P"], c["K"], c["N"], c["V"], c["S"], c["M"], c["A"], c["D"]
    table = {
        "k_bilateral_outlier": 4 * P + 2 * K * c["valid"],
        "k_erode_normals_radii": 2 * P + 2 * P + 8 * P + 4 * c["valid"] + 20 * P,
        "k_project": 16 * N + 16 * V,
        "k_associate": 16 * V + 16 * V + 1.5 * V * (2 + 4 + 8) + 12 * S_,
        "k_merge": 16 * V + 4 * V + 1.5 * V * (2 + 4 + 4),
        "k_blend": 2 * P + 4 * P + 2 * P,
        # list entry + merge flag + 11 surfel rows read per visible surfel, rasters of <= 2 pixels; only the D
        # surfels the frame really changes are written back (11 rows)
        "k_integrate": 16 * V + V + 44 * V + 1.5 * V * 29 + 44 * D,
        "k_update_neighbors": 4 * V + 36 * V + 4 * 16 * V,
        "k_new_surfel_scan": 2 * P + 8 * P + P + 4 * P,
        "k_create_surfels": 5 * P + 72 * M,
        "k_reg_accumulate": 16 * N + 16 * N + 32 * A,
        "k_reg_step": (4 + 16 + 12 + 12) * N + (52 + 12 * 4 + 16) * A,
    }
    return float(table.get(kernel, 0.0))


def cpu_baseline(stream, pp, ip, cam, rows, frame, budget_s=24.0, runs=3, max_frames=12):
    """CPU walk (oracle/cpu_walk.c) of the per-pixel filter chain + the per-surfel min-depth /
    association loop on a bounded sample of the stream: one untimed warm-up pass, then `runs` timed
    passes over the same frames; value = median, spread reported. Threads pinned (OMP_PROC_BIND=close)."""
    from oracle import cpu_walk
    depth = stream.depth.cpu().numpy()
    K = pp.outlier_filtering_frame_count
    threads = cpu_walk.max_threads()
    first, last = stream.integrated_range()
    frames = list(range(first, last))[:max_frames]

    def one_pass(limit_s):
        t0 = time.perf_counter()
        done = 0
        for f in frames:
            others = [depth[f - (i + 1)] for i in range(K // 2)] + [depth[f + (i + 1)] for i in range(K // 2)]
            d, n, r = cpu_walk.preprocess(pp, cam.fx, cam.fy, cam.cx, cam.cy, depth[f], others,
                                          stream.others_TR_reference[f])
            cpu_walk.associate(rows, frame, cam.fx, cam.fy, cam.cx, cam.cy, stream.frame_T_global[f], d, n,
                               ip.sensor_noise_factor, ip.normal_compatibility_threshold_deg, ip.depth_scaling)
            done += 1
            if time.perf_counter() - t0 > limit_s:
                break
        return done, time.perf_counter() - t0

    done, _ = one_pass(budget_s / (runs + 1))          # warm-up: page in the arrays, spin up the thread pool
    frames = frames[:done]
    rates = []
    for _ in range(runs):
        n_done, dt = one_pass(1e9)
        rates.append(n_done / dt)
    rates.sort()
    return {"value": rates[len(rates) // 2], "unit": "frames/s", "cores": threads, "kind": "port",
            "runs": rates, "spread": (rates[-1] - rates[0]) / rates[len(rates) // 2],
            "sample": f"median of {runs} warmed passes over {len(frames)} frames of the same stream (threads pinned): "
                      f"a1-a5 per pixel + min-depth/association (a7/a8) over the final cloud of {rows.shape[1]} surfels; "
                      f"merge/blend/integrate/neighbours/creation/regularisation are NOT walked (the reference has "
                      f"no CPU Integrate)"}


DUMP_PROBES = 1 << 18   # 9.4 MB of dumped arrays, well inside the 64 MB budget


def probe_points(stream, first, last, count):
    """`count` fixed points on the scene's surfaces, a function of the seeded input stream only: pixels with a
    measurement, drawn with a fixed seed from the integrated frames and unprojected with their frames' poses."""
    rng = np.random.default_rng(0)
    cam, frames, height, width = stream.camera, stream.depth.shape[0], stream.depth.shape[1], stream.depth.shape[2]
    f = rng.integers(first, min(last, frames), 4 * count)
    v = rng.integers(0, height, 4 * count)
    u = rng.integers(0, width, 4 * count)
    index = [torch.from_numpy(i).to(stream.depth.device) for i in (f, v, u)]
    # (gathered as int16: CUDA has no uint16 gather)
    z = stream.depth.view(torch.int16)[tuple(index)].cpu().numpy().view(np.uint16).astype(np.float64)
    keep = np.flatnonzero(z > 0)[:count]
    f, v, u, z = f[keep], v[keep], u[keep], z[keep] / stream.depth_scaling
    local = np.stack([(u + 0.5 - cam.cx) / cam.fx * z, (v + 0.5 - cam.cy) / cam.fy * z, z], axis=1)
    pose = stream.global_T_frame[f].astype(np.float64)
    return np.einsum("nij,nj->ni", pose[:, :, :3], local) + pose[:, :, 3]


def dump_outputs(out_dir, rec, stats, stream, first, last):
    """What a caller of the timed path receives after a step: the CUDASurfelBuffersCPU arrays of the cloud
    (TransferAllToCPU at the step's last frame) and the step's counts.

    The slot order of the cloud is not reproducible (which of several supporting surfels wins a pixel feeds back
    into how many surfels each frame creates, and float atomics round differently from run to run), so the rows
    are sampled by place, not by slot: for each of DUMP_PROBES fixed points on the scene's surfaces
    (probe_points), the row of the nearest surfel that is not merged away. Every file has the same shape from run
    to run and from build to build. Stamps are written as float64 (exact)."""
    from scipy.spatial import cKDTree
    out_dir.mkdir(parents=True, exist_ok=True)
    buffers = rec.TransferAllToCPU(None, last - 1)
    n = int(buffers["surfel_count"])
    arrays = {k: (v[:n].astype(np.float64) if v.dtype == np.uint32 else v[:n])
              for k, v in buffers.items() if k.endswith("_buffer")}
    live = np.flatnonzero(arrays["surfel_radius_squared_buffer"] >= 0)
    probes = probe_points(stream, first, last, DUMP_PROBES)
    if len(live):
        xyz = np.stack([arrays[f"surfel_{c}_buffer"][live] for c in "xyz"], axis=1).astype(np.float64)
        _, nearest = cKDTree(xyz).query(probes)
        rows = live[nearest]
        sampled = {k: a[rows] for k, a in arrays.items()}
    else:
        sampled = {k: np.full(len(probes), np.nan, dtype=a.dtype) for k, a in arrays.items()}
    sampled["stream_counts"] = np.array([stats.frames_integrated, stats.surfels_size, stats.surfel_count],
                                        dtype=np.float64)
    for name, a in sampled.items():
        np.save(out_dir / f"{name}.npy", a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="product", choices=["product", "reference"])
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--cap", type=int, default=5_000_000)
    ap.add_argument("--sigma-depth", type=float, default=None)
    ap.add_argument("--required-inliers", type=int, default=-1,
                    help="outlier_filtering_required_inliers (-1 = all 8 other frames, the reference's default)")
    ap.add_argument("--erosion-radius", type=int, default=2, help="depth_erosion_radius (reference default 2)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-roofline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step computed as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1 (the timed steps are what the line reports and --dump-outputs writes)")
    warmup = max(args.warmup, 3)

    # stdout carries exactly one JSON line: NCCL's version banner (NCCL_DEBUG=VERSION) goes to stdout too
    if os.environ.get("NCCL_DEBUG", "").upper() == "VERSION":
        os.environ["NCCL_DEBUG"] = "WARN"
    info = D.rank_info_from_env()
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the surfel kernels have no CPU fallback")
    device = torch.device("cuda", info.local_rank)
    torch.cuda.set_device(device)
    D.init_process_group(info, backend="nccl")

    lib = _lib.load_product() if args.impl == "product" else _lib.load_reference_oracle()
    cam = S.Camera.tum(args.width, args.height)
    stream = S.make_stream(cam, args.frames, stream_id=info.rank, sigma_depth=args.sigma_depth, device=device)
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    pp.outlier_filtering_required_inliers = args.required_inliers
    pp.depth_erosion_radius = args.erosion_radius
    ip = IntegrateParams.defaults()
    first, last = stream.integrated_range()
    frames_per_step = last - first
    rec = R.CUDASurfelReconstruction(args.cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=lib)
    launches_per_step = [0]

    def step_device():
        rec.reset()
        st = rec.stream_run(None, stream.depth, stream.color, stream.global_T_frame, stream.frame_T_global,
                            stream.others_TR_reference, pp, ip, first, last)
        launches_per_step[0] = int(st.kernel_launches)
        return st

    # ---- value: frames resident in HBM ----
    with ClockSampler(info.local_rank) as clocks:
        ms, stats = timed_steps(info, device, step_device, warmup, args.steps)
    ms_max, frames_total = D.aggregate(info, ms, frames_per_step * args.steps, device)
    ms_per_rank = D.gather_values(info, ms / args.steps, device)
    value = frames_total / (ms_max * 1e-3)
    if args.dump_outputs and info.rank == 0:
        dump_outputs(Path(args.dump_outputs), rec, stats, stream, first, last)

    # ---- e2e: host (pinned) frames in, CUDASurfelBuffersCPU arrays out ----
    host_depth = stream.depth.cpu().pin_memory()
    host_color = stream.color.cpu().pin_memory()
    n_final = int(stats.surfels_size)
    host_buffers = {k: torch.empty(max(n_final * 2, 1), dtype=torch.int32 if "stamp" in k else torch.float32
                                   ).pin_memory().numpy().view(np.uint32 if "stamp" in k else np.float32)
                    for k in ["surfel_x_buffer", "surfel_y_buffer", "surfel_z_buffer", "surfel_radius_squared_buffer",
                              "surfel_normal_x_buffer", "surfel_normal_y_buffer", "surfel_normal_z_buffer",
                              "surfel_last_update_stamp_buffer"]}
    io_bytes = [0, 0]

    def step_host():
        rec.reset()
        st = rec.stream_run(None, host_depth, host_color, stream.global_T_frame, stream.frame_T_global,
                            stream.others_TR_reference, pp, ip, first, last)
        out = rec.TransferAllToCPU(None, last - 1, host_buffers)
        io_bytes[0] = int(st.h2d_bytes)
        io_bytes[1] = int(st.d2h_bytes) + 8 * 4 * int(out["surfel_count"])
        return st

    e2e_steps = max(1, min(args.steps, 5))
    ms_e2e, _ = timed_steps(info, device, step_host, 1, e2e_steps)
    ms_e2e_max, frames_e2e = D.aggregate(info, ms_e2e, frames_per_step * e2e_steps, device)
    e2e_value = frames_e2e / (ms_e2e_max * 1e-3)

    # ---- roofline: profiled extra pass (product only; per-kernel events inside the library) ----
    roofline = None
    kernel_table = None
    if args.impl == "product" and info.rank == 0 and not args.no_roofline:
        peak, peak_src = measured_peaks()
        # The roofline region is the LAST `tail` frames of a step: there the cloud is at its final size, so the
        # algorithmic bytes (counters of the last frame) and the mean launch durations (per-kernel CUDA events on
        # the launching stream) describe the same work. (Over the whole step the cloud grows from 0 to N: bytes of
        # the last frame over the mean duration of all frames would overstate the bandwidth.)
        tail = min(40, frames_per_step)
        rec.reset()
        if last - tail > first:
            rec.stream_run(None, stream.depth, stream.color, stream.global_T_frame, stream.frame_T_global,
                           stream.others_TR_reference, pp, ip, first, last - tail)
        lib.call("profile_kernels", 1)
        rec.stream_run(None, stream.depth, stream.color, stream.global_T_frame, stream.frame_T_global,
                       stream.others_TR_reference, pp, ip, last - tail, last)
        nk = lib.fn["profile_kernel_count"]()
        tot = (torch.zeros(nk, dtype=torch.float64).numpy())
        cnt = np.zeros(nk, dtype=np.uint64)
        import ctypes as C
        lib.call("profile_report", tot.ctypes.data_as(C.POINTER(C.c_double)), cnt.ctypes.data_as(C.POINTER(C.c_uint64)), nk)
        lib.call("profile_kernels", 0)
        fc = (C.c_uint64 * 4)()
        lib.call("frame_counters", rec._h, None, C.byref(fc))
        rows_now, n_now, _ = rec.dump_state()
        stamps = rows_now[18].view(np.uint32)
        counters = {"P": cam.width * cam.height, "K": pp.outlier_filtering_frame_count,
                    "valid": int((stream.depth[last - 1].to(torch.int32) > 0).sum()), "N": int(fc[0]), "V": int(fc[1]),
                    "S": int(fc[2]), "M": int(fc[3]),
                    "A": int((stamps.astype(np.int64) >= (last - 1) - ip.regularization_frame_window_size).sum()),
                    "D": int((stamps == np.uint32(last - 1)).sum())}
        kernel_table = {}
        total_ms = float(tot.sum())
        for i in range(nk):
            if cnt[i]:
                name = lib.fn["profile_kernel_name"](i).decode()
                kernel_table[name] = {"launches": int(cnt[i]), "mean_us": tot[i] / cnt[i] * 1e3,
                                      "share": tot[i] / total_ms}
        roofline = {"bound": "hbm", "peak": peak, "unit": "GB/s", "peak_source": peak_src, "counters": counters,
                    "region": f"last {tail} frames of a step"}
        # The same kernels as they run inside the frame graph: start / end stamps written by the kernels
        # themselves (sm_timeline_enable), mean over the same last frames of a full step.
        frames_pow2 = 1 << (args.frames - 1).bit_length()
        lib.call("timeline_enable", rec._h, frames_pow2)
        step_device()
        stamps_buf = np.zeros((frames_pow2, nk, 2), dtype=np.uint64)
        lib.call("timeline_read", rec._h, stamps_buf.ctypes.data_as(C.POINTER(C.c_uint64)), frames_pow2)
        lib.call("timeline_enable", rec._h, 0)
        launched = stamps_buf[:, :, 0] != np.uint64(0xFFFFFFFFFFFFFFFF)
        in_region = np.zeros(frames_pow2, dtype=bool)
        in_region[[f % frames_pow2 for f in range(last - tail, last)]] = True
        launched &= in_region[:, None]
        for i in range(nk):
            name = lib.fn["profile_kernel_name"](i).decode()
            if launched[:, i].any():
                dur = (stamps_buf[:, i, 1].astype(np.float64) - stamps_buf[:, i, 0].astype(np.float64))[launched[:, i]]
                kernel_table.setdefault(name, {})["pipelined_us"] = float(dur.mean() / 1e3)
        project = [i for i in range(nk) if lib.fn["profile_kernel_name"](i).decode() == "k_project"][0]
        starts = np.sort(stamps_buf[launched[:, project], project, 0].astype(np.float64))
        if len(starts) > 2:
            roofline["pipelined_frame_period_us"] = float(np.median(np.diff(starts)) / 1e3)
        # The dominant kernel is the longest one ON THE DEPENDENCY CYCLE THAT BOUNDS THE FRAME RATE, as the
        # kernels run inside the pipeline (device timeline) - not the largest share of the serial,
        # host-launch-bound event pass, where a kernel off the critical path can look dominant.
        cycles = {"integrate->update_neighbors->reg_accumulate->reg_step":
                  ["k_integrate", "k_update_neighbors", "k_reg_accumulate", "k_reg_step"],
                  "integrate->create->project_tail->associate->blend":
                  ["k_integrate", "k_create_surfels", "k_project_tail" if "k_project_tail" in kernel_table else "k_project",
                   "k_associate", "k_blend"]}
        cycle_us = {name: sum(kernel_table.get(k, {}).get("pipelined_us", 0.0) for k in ks) for name, ks in cycles.items()}
        binding = max(cycle_us, key=cycle_us.get)
        dom = max((k for k in cycles[binding] if "mean_us" in kernel_table.get(k, {})),
                  key=lambda k: kernel_table[k].get("pipelined_us", 0.0))
        # Algorithmic bytes use the LAST frame's counters (largest cloud of the step); the mean launch
        # duration (CUDA events on the launching stream, serial pass) is over the whole step: conservative.
        b = algorithmic_bytes(dom, counters)
        dur = kernel_table[dom]["mean_us"] * 1e-6
        achieved = b / dur / 1e9
        roofline.update({"kernel": dom, "achieved": achieved, "frac": achieved / peak,
                         "algorithmic_bytes_per_launch": b, "mean_launch_us": kernel_table[dom]["mean_us"],
                         "pipelined_launch_us": kernel_table[dom].get("pipelined_us"),
                         "achieved_pipelined": b / (kernel_table[dom].get("pipelined_us", float("nan")) * 1e-6) / 1e9,
                         "share_of_step": kernel_table[dom]["share"], "binding_cycle": binding, "cycle_us": cycle_us})
        for name in ("k_bilateral_outlier", "k_associate"):
            if name in kernel_table:
                bb = algorithmic_bytes(name, counters)
                kernel_table[name]["achieved_gbs"] = bb / (kernel_table[name]["mean_us"] * 1e-6) / 1e9
                kernel_table[name]["frac_of_hbm_peak"] = kernel_table[name]["achieved_gbs"] / peak

    # ---- cpu baseline (rank 0, N = 1, product arm) ----
    cpu = None
    if info.rank == 0 and info.world_size == 1 and not args.no_cpu_baseline:
        if args.impl == "product":
            rows, _, _ = rec.dump_state()
            cpu = cpu_baseline(stream, pp, ip, cam, rows, last - 1)
        else:
            cpu = {"value": value, "unit": "frames/s", "cores": 1, "kind": "reference",
                   "sample": "full workload; the reference implements this path only as CUDA kernels, so its arm "
                             "runs them (rebuilt unmodified for sm_90a) on the same GPU, driven by one host thread"}

    if info.rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": info.world_size, "steps": args.steps,
            "warmup": warmup, "ms_per_step": ms_max / args.steps, "ms_per_step_per_rank": ms_per_rank,
            "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"synthetic TUM-fr1/desk-shaped {cam.width}x{cam.height} stream, {args.frames} "
                                   f"frames ({frames_per_step} integrated) per GPU, full preprocess + Integrate(), "
                                   f"{args.cap} surfel cap" + (", one independent stream per GPU" if info.world_size > 1 else ""),
                       "frames_per_step": frames_per_step, "surfels_after_step": int(stats.surfels_size),
                       "l2": f"inputs larger than L2 ({stream.depth.numel() * 2 + stream.color.numel():,} B of frames per "
                             f"step), no flush",
                       "required_inliers": args.required_inliers, "erosion_radius": args.erosion_radius,
                       "sigma_depth": args.sigma_depth},
            "clocks": clocks.summary(),
            "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": io_bytes[0],
                    "d2h_bytes_per_step": io_bytes[1], "steps": e2e_steps},
            "gpu_launches": launches_per_step[0] * args.steps,
        }
        if args.impl == "reference":
            line["impl"] = "reference"
        if roofline:
            line["roofline"] = roofline
            line["kernels"] = kernel_table
        if cpu:
            line["cpu_baseline"] = cpu
        print(json.dumps(line))
    if info.is_distributed:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
