"""BASELINE config 1 at scale: one meshing iteration of the reference's own CPU meshing (oracle/_ref/libmeshing_ref.so:
IntegrateCUDABuffers -> CheckRemeshing -> Triangulate over N fresh surfels of a surface) with its octree answering the
neighbour queries, and with ONE sm_knn_query batch answering them (DESIGN.md section 5.4). Prints one JSON object with
the CPU times of both runs, the GPU time of the batch end to end (host arrays in, host arrays out), and whether the
two meshes are identical.

    python tools/meshing_probe.py --points 1000000 --out probe_out/meshing_probe.json
"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import meshing_ref  # noqa: E402  (the reference's CPU meshing is the thing being fed here)
from surfelmeshing_b200.knn import SurfelKnnIndex  # noqa: E402
from tests import knn_cases  # noqa: E402


def run(cloud, batch):
    m = meshing_ref.SurfelMeshing()
    t0 = time.perf_counter()
    m.integrate(1, **cloud)
    t1 = time.perf_counter()
    if batch is not None:
        m.set_knn_batch(*batch)
    t2 = time.perf_counter()
    m.check_remeshing()
    t3 = time.perf_counter()
    m.triangulate()
    t4 = time.perf_counter()
    tri, stats = m.triangles(), m.query_stats()
    m.close()
    return tri, {"integrate_s": t1 - t0, "check_remeshing_s": t3 - t2, "triangulate_s": t4 - t3,
                 "total_s": (t1 - t0) + (t3 - t2) + (t4 - t3)}, stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.points
    spacing = 1.0 / np.sqrt(n)
    cloud = knn_cases.meshing_cloud(n, 6, "sheet", thickness=0.5 * spacing)
    tri, cpu_times, stats = run(cloud, None)

    f = meshing_ref.SurfelMeshing.MAX_NEIGHBOR_SEARCH_RANGE_INCREASE_FACTOR
    r2 = (cloud["radius_squared"] * np.float32(f * f)).astype(np.float32)
    dev = torch.device("cuda:0")
    pin = lambda v: torch.from_numpy(np.ascontiguousarray(v)).pin_memory()
    hx, hy, hz, hr2, hrad = [pin(cloud[k]) for k in ("x", "y", "z")] + [pin(r2), pin(cloud["radius_squared"])]
    out_d2 = torch.empty((n, 64), dtype=torch.float32).pin_memory()
    out_idx = torch.empty((n, 64), dtype=torch.int32).pin_memory()
    out_cnt = torch.empty((n,), dtype=torch.int32).pin_memory()
    index = SurfelKnnIndex(n)
    gpu_s = []
    for rep in range(4):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gx, gy, gz, gr2, grad = [v.to(dev, non_blocking=True) for v in (hx, hy, hz, hr2, hrad)]
        index.build(gx, gy, gz, 2.0 * float(np.sqrt(r2.max())), radius_squared=grad)
        d2, idx, cnt = index.FindNearestSurfelsWithinRadius(gx, gy, gz, gr2, 64)
        out_d2.copy_(d2, non_blocking=True)
        out_idx.copy_(idx, non_blocking=True)
        out_cnt.copy_(cnt, non_blocking=True)
        torch.cuda.synchronize()
        if rep:
            gpu_s.append(time.perf_counter() - t0)
    # the same through the host-array entry point of the C ABI (pageable numpy arrays in and out)
    host_s = []
    host_out = (np.zeros((n, 64), np.float32), np.zeros((n, 64), np.uint32), np.zeros((n,), np.int32))   # reused, already touched
    for rep in range(4):
        t0 = time.perf_counter()
        hd2, hidx, hcnt = index.batch_host(cloud["x"], cloud["y"], cloud["z"], cloud["radius_squared"], float(f * f), 64, out=host_out)
        if rep:
            host_s.append(time.perf_counter() - t0)
    assert np.array_equal(hcnt, out_cnt.numpy()) and np.array_equal(hidx, out_idx.numpy().view(np.uint32))
    batch = (out_d2.numpy(), out_idx.numpy().view(np.uint32), out_cnt.numpy(), r2)
    tri_fed, fed_times, fed_stats = run(cloud, batch)
    result = {"workload": f"{n} fresh surfels on a sheet, radius 1.5 x spacing, one meshing iteration of the reference's CPU code",
              "triangles": int(len(tri)), "identical_mesh": bool(np.array_equal(tri, tri_fed)),
              "octree": cpu_times, "octree_queries": int(stats[1]),
              "gpu_batch": fed_times, "queries_answered_from_the_batch": int(fed_stats[0]), "queries_left_to_the_octree": int(fed_stats[1]),
              "gpu_batch_end_to_end_s": float(np.median(gpu_s)),
              "gpu_batch_host_api_s": float(np.median(host_s)),
              "mean_neighbours_in_batch_row": float(out_cnt.numpy().mean())}
    result["iteration_speedup"] = cpu_times["total_s"] / (fed_times["total_s"] + result["gpu_batch_end_to_end_s"])
    result["iteration_speedup_host_api"] = cpu_times["total_s"] / (fed_times["total_s"] + result["gpu_batch_host_api_s"])
    print(json.dumps(result))
    if a.out:
        Path(a.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
