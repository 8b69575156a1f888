"""Writes tests/golden/knn_golden.npz: answers of the REFERENCE's CPU octree (oracle/_ref/liboctree_ref.so, i.e.
applications/surfel_meshing/src/surfel_meshing/octree.cc compiled by oracle/Makefile) for the seeded cases of
tests/knn_cases.py. Run where the reference sources are present (oracle/Makefile: REF builds the oracle):

    make -C oracle ref && python tests/golden/make_knn_golden.py
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from oracle import octree_ref  # noqa: E402
from tests import knn_cases  # noqa: E402


def main():
    out = {}
    for name, (x, y, z), r2_value, k in (
            ("random", knn_cases.random_cloud(4000, 11), 1.5 ** 2, 16),
            ("nasty", knn_cases.nasty_cloud(300, 12), 0.35 ** 2, 6),
            ("surface", knn_cases.surface_cloud(6000, 13), 0.07 ** 2, 64)):
        n = len(x)
        state = knn_cases.states(n, 14)
        rng = np.random.default_rng(15)
        qi = rng.integers(0, n, 300)
        r2 = np.full(len(qi), r2_value, np.float32)
        for label, ic, fr in (("all", 1, 1), ("triangulate", 0, 1), ("remesh", 1, 0)):
            tree = octree_ref.Octree(x, y, z, state)
            d2, idx, cnt, _ = tree.query(x[qi], y[qi], z[qi], r2, k, ic, fr)
            tree.close()
            out[f"{name}_{label}_d2"], out[f"{name}_{label}_idx"], out[f"{name}_{label}_cnt"] = d2, idx, cnt
        out[f"{name}_query_index"] = qi
    np.savez_compressed(ROOT / "tests" / "golden" / "knn_golden.npz", **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
