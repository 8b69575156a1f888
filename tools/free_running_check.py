"""Free-running totals of a whole stream: the product under candidate supporting-surfel rules against several runs of
the reference's kernels (oracle/_ref), in units of the oracle's own run-to-run spread.

    python tools/free_running_check.py --width 1280 --height 960 --frames 1000 --cap 20000000 \\
        --rule default --rule 303104,0.02,0.25,32 --out probe_out/free_hd.json
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from surfelmeshing_b200 import _lib, reconstruction as R, synthetic as S  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--cap", type=int, default=5_000_000)
    ap.add_argument("--oracle-runs", type=int, default=3)
    ap.add_argument("--rule", action="append", default=[], help="'default' or wave,early,index_order,lanes[,phase[,early_later[,index_order_later[,early_second]]]]")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cam = S.Camera.tum(a.width, a.height)
    st = S.make_stream(cam, a.frames, device="cuda")
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    first, last = st.integrated_range()

    def run(rec):
        rec.reset()
        s = rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip, first, last)
        return [int(s.surfels_size), int(s.surfel_count), int(s.surfels_size) - int(s.surfel_count)]

    ref = R.CUDASurfelReconstruction(a.cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=_lib.load_reference_oracle())
    oracle = np.array([run(ref) for _ in range(a.oracle_runs)])
    ref.close()
    mean, spread = oracle.mean(axis=0), oracle.max(axis=0) - oracle.min(axis=0)
    result = {"config": vars(a), "oracle_runs": oracle.tolist(), "oracle_mean": mean.tolist(), "oracle_spread": spread.tolist(), "rules": {}}
    print("oracle [slots, live, merged]:", oracle.tolist(), "spread", spread.tolist())
    rec = R.CUDASurfelReconstruction(a.cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy)
    for rule in a.rule or ["default"]:
        if rule != "default":
            # wave,early,index_order,lanes[,phase[,early_later[,index_order_later[,early_second]]]]
            parts = rule.split(",")
            wave, early, index_order, lanes, phase, early_later, index_later, early_second = \
                [float(v) for v in parts] + [0.0, -1.0, -1.0, -1.0][len(parts) - 4:]
            rec.configure("tiebreak_wave_offset", phase)
            rec.configure("tiebreak_lanes", lanes)
            rec.configure("tiebreak_wave", wave)
            rec.configure("tiebreak_early_fraction", early)
            rec.configure("tiebreak_index_order_fraction", index_order)
            rec.configure("tiebreak_early_fraction_later", early_later)
            rec.configure("tiebreak_index_order_fraction_later", index_later)
            rec.configure("tiebreak_early_fraction_second", early_second)
        got = np.array(run(rec))
        dev = (got - mean) / np.maximum(spread, 1)
        result["rules"][rule] = {"totals": got.tolist(), "deviation_in_oracle_spreads": dev.tolist(),
                                 "relative": ((got - mean) / mean).tolist()}
        print(f"{rule:28s} {got.tolist()}  deviation / spread {np.round(dev, 2).tolist()}  relative {np.round(100 * (got - mean) / mean, 3).tolist()} %")
    rec.close()
    if a.out:
        Path(a.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
