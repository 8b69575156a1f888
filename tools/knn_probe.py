"""Neighbour search for the meshing thread (SURVEY section 8 f4): GPU batch (libsurfel_b200.so, sm_knn_*) against the
reference's own CPU octree (oracle/_ref/liboctree_ref.so) on a synthetic surfel sheet.

    python tools/knn_probe.py --points 1000000 --queries 1000000 --out probe_out/knn_probe.json

Prints one JSON object: build time, queries/s with everything resident in HBM (CUDA events), queries/s end to end
(host arrays in, host arrays out, pinned staging, copies inside the timed region), the reference octree's queries/s
on one host thread over a bounded sample (the meshing thread's pattern: the non-passive query is not thread safe),
and a parity check of that sample.
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

from oracle import octree_ref  # noqa: E402  (reference leg only)
from surfelmeshing_b200.knn import SurfelKnnIndex  # noqa: E402
from tests import knn_cases  # noqa: E402
from tests.test_octree_oracle import assert_same_neighbours  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=64)
    ap.add_argument("--spacing", type=float, default=0.005)
    ap.add_argument("--radius-factor", type=float, default=2.5, help="query radius in units of the point spacing")
    ap.add_argument("--cell-factor", type=float, default=2.0, help="cell size in units of the query radius")
    ap.add_argument("--cpu-sample", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cloud", default="sheet", choices=["sheet", "random"],
                    help="sheet: a surfel surface; random: uniform points in a cube (BASELINE config 1: the pattern of the "
                         "reference's octree / triangulation tests), spacing = mean distance to the nearest neighbour")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    if a.cloud == "random":
        extent = 0.5 * a.spacing * (a.points ** (1.0 / 3.0)) / 0.554   # nearest-neighbour distance of a Poisson cloud
        x, y, z = knn_cases.random_cloud(a.points, 7, extent=extent)
    else:
        x, y, z = knn_cases.surface_cloud(a.points, 7, spacing=a.spacing)
    rng = np.random.default_rng(8)
    qi = rng.permutation(a.points)[: a.queries] if a.queries <= a.points else rng.integers(0, a.points, a.queries)
    radius = a.radius_factor * a.spacing
    r2 = np.full(len(qi), radius * radius, np.float32)
    qx, qy, qz = x[qi], y[qi], z[qi]
    cell = a.cell_factor * radius

    dev = torch.device("cuda:0")
    dx, dy, dz = [torch.from_numpy(v).to(dev) for v in (x, y, z)]
    dqx, dqy, dqz, dr2 = [torch.from_numpy(v).to(dev) for v in (qx, qy, qz, r2)]
    index = SurfelKnnIndex(a.points)
    ev = lambda: torch.cuda.Event(enable_timing=True)

    build_ms, query_ms = [], []
    for rep in range(a.reps + 2):
        e0, e1, e2 = ev(), ev(), ev()
        e0.record()
        index.build(dx, dy, dz, cell)
        e1.record()
        d2, idx, cnt = index.FindNearestSurfelsWithinRadius(dqx, dqy, dqz, dr2, a.k)
        e2.record()
        torch.cuda.synchronize()
        if rep >= 2:
            build_ms.append(e0.elapsed_time(e1))
            query_ms.append(e1.elapsed_time(e2))
    found = cnt.cpu().numpy()

    # end to end: host arrays -> pinned -> device, build + query, results back to pinned host memory
    pin = lambda v: torch.from_numpy(v).pin_memory()
    hx, hy, hz, hqx, hqy, hqz, hr2 = [pin(v) for v in (x, y, z, qx, qy, qz, r2)]
    out_d2 = torch.empty((len(qi), a.k), dtype=torch.float32).pin_memory()
    out_idx = torch.empty((len(qi), a.k), dtype=torch.int32).pin_memory()
    out_cnt = torch.empty((len(qi),), dtype=torch.int32).pin_memory()
    e2e_s = []
    for rep in range(a.reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gx, gy, gz, gqx, gqy, gqz, gr2 = [v.to(dev, non_blocking=True) for v in (hx, hy, hz, hqx, hqy, hqz, hr2)]
        index.build(gx, gy, gz, cell)
        d2, idx, cnt = index.FindNearestSurfelsWithinRadius(gqx, gqy, gqz, gr2, a.k)
        out_d2.copy_(d2, non_blocking=True)
        out_idx.copy_(idx, non_blocking=True)
        out_cnt.copy_(cnt, non_blocking=True)
        torch.cuda.synchronize()
        if rep >= 1:
            e2e_s.append(time.perf_counter() - t0)

    result = {
        "workload": f"{a.points} surfels {'on a sheet' if a.cloud == 'sheet' else 'uniform in a cube'} (spacing {a.spacing} m), {len(qi)} queries, radius {radius:.4f} m, "
                    f"k <= {a.k}, cell {cell:.4f} m",
        "mean_neighbours_found": float(found.mean()), "queries_at_cap": float((found == a.k).mean()),
        "build_ms": float(np.median(build_ms)), "query_ms": float(np.median(query_ms)),
        "queries_per_s_resident": len(qi) / (np.median(query_ms) * 1e-3),
        "queries_per_s_resident_incl_build": len(qi) / ((np.median(query_ms) + np.median(build_ms)) * 1e-3),
        "queries_per_s_e2e": len(qi) / float(np.median(e2e_s)),
        "e2e_h2d_bytes": int(4 * (3 * a.points + 4 * len(qi))), "e2e_d2h_bytes": int(len(qi) * (8 * a.k + 4)),
        # bytes one query cannot avoid: its own record, the records inside the ball, its outputs
        "algorithmic_bytes_per_query": float(16 + 16 * found.mean() + 8 * a.k + 4),
    }
    result["achieved_GBps"] = result["algorithmic_bytes_per_query"] * result["queries_per_s_resident"] / 1e9

    if octree_ref.available():
        m = min(a.cpu_sample, len(qi))
        t0 = time.perf_counter()
        tree = octree_ref.Octree(x, y, z)
        build_s = time.perf_counter() - t0
        want_d2, want_idx, want_cnt, seconds = tree.query(qx[:m], qy[:m], qz[:m], r2[:m], a.k)
        tree.close()
        got = (out_d2.numpy()[:m], out_idx.numpy()[:m].view(np.uint32), out_cnt.numpy()[:m])
        assert_same_neighbours(got, (want_d2, want_idx, want_cnt), a.k)
        result["reference_octree"] = {"kind": "reference", "cores": 1, "sample": f"first {m} queries, one thread",
                                      "build_s": build_s, "queries_per_s": m / seconds, "parity_checked_queries": m}
        result["speedup_e2e_vs_reference_octree"] = result["queries_per_s_e2e"] / (m / seconds)
    print(json.dumps(result))
    if a.out:
        Path(a.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
