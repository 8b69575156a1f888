#!/usr/bin/env python
"""Writes tests/golden/oracle_answers.json: what the REFERENCE's own kernels (oracle/_ref/libsurfel_ref.so)
answer on the seeded inputs of the parity tests that compare the product with them, so that those tests
run without the reference tree. Bit-exact answers are stored as sha256 digests (tests/util.py: digest),
counts as numbers; every entry also holds the digest of its input (depth stream or surfel state), which the
tests check first. The smooth positions after Regularize(), compared with a tolerance, go to
oracle_regularized_smooth.npz.xz beside the JSON file. Run on a GPU with the oracle built:

    python tests/golden/make_oracle_answers.py [output.json]
"""
import io
import json
import lzma
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
from surfelmeshing_b200 import _lib  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from tests import test_parity_gpu as P  # noqa: E402
from tests import test_round2_gpu as Q  # noqa: E402
from tests.util import SMOOTH_ROWS, digest, load_golden  # noqa: E402


def main(out_path):
    ref = _lib.load_reference_oracle()
    out = {}
    for width, height in P.RAGGED_SIZES:
        cam, pp, raw, others, mats, inputs = P.ragged_case(width, height)
        out[f"preprocess/{width}x{height}"] = dict(P.stage_digests(P.run_stages(ref, cam, pp, raw, others, mats)),
                                                   inputs=inputs)
    for variant in P.PREPROCESS_VARIANTS:
        cam, pp, raw, others, mats, inputs = P.variant_case(variant)
        out[f"preprocess_variant/{variant}"] = dict(P.stage_digests(P.run_stages(ref, cam, pp, raw, others, mats)),
                                                    inputs=inputs)
    for sigma in P.FULL_SIZE_SIGMAS:
        cam, st, pp, ip = P.full_size_case(sigma)
        first, last = st.integrated_range()
        rec = R.CUDASurfelReconstruction(2_000_000, 640, 480, cam.fx, cam.fy, cam.cx, cam.cy, lib=ref)
        s = rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                           ip, first, last)
        out[f"full_size/{sigma}"] = {"inputs": digest(st.depth.cpu().numpy()), "stream": P.stream_counts(s)}
        rec.close()
    cam, st, pp, ip, cap = P.large_frame_case()
    first, last = st.integrated_range()
    rec = R.CUDASurfelReconstruction(cap, cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, lib=ref)
    s1 = rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                        first, first + 1)
    rows, n, _ = rec.dump_state()
    entry = {"inputs": digest(st.depth.cpu().numpy()),
             "first_frame": {"surfels_size": int(s1.surfels_size), "rows": P.first_frame_row_digests(rows, n)}}
    rec.reset()
    s = rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                       first, last)
    entry["stream"] = P.stream_counts(s)
    out["large_frame"] = entry
    rec.close()
    # The oracle's free-running totals vary more between processes than within one, and the test runs the product
    # in a process of its own: every run of the envelope comes from a separate process.
    runs = [json.loads(subprocess.run([sys.executable, __file__, "--free-running-run"], check=True, capture_output=True,
                                      text=True).stdout.strip().splitlines()[-1]) for _ in range(6)]
    out["free_running"] = {"inputs": runs[0]["inputs"], "runs": [r["totals"] for r in runs]}
    assert all(r["inputs"] == runs[0]["inputs"] for r in runs)
    runs = out["free_running"]["runs"]
    # hand-off and visualisation sweeps on the reference's state after the golden frames
    golden = load_golden()
    rows, n, merges, last = P.golden_final_state(golden)
    rec = P.golden_reconstruction(golden, lib=ref)
    rec.load_state(rows, merges)
    handoff, _, _ = P.handoff_outputs(rec, last, n)
    ip = P.IntegrateParams.defaults()
    rec.Regularize(None, last, ip.regularizer_weight, ip.radius_factor_for_regularization_neighbors,
                   ip.regularization_frame_window_size)
    torch.cuda.synchronize()
    regularized = rec.dump_state()[0]
    out["golden_handoff"] = {"inputs": digest(rows), "handoff": handoff,
                             "regularized_rows": P.regularized_row_digests(regularized)}
    buf = io.BytesIO()
    np.savez(buf, smooth=np.ascontiguousarray(regularized[list(SMOOTH_ROWS)]))
    (Path(out_path).parent / "oracle_regularized_smooth.npz.xz").write_bytes(
        lzma.compress(buf.getvalue(), preset=9 | lzma.PRESET_EXTREME))
    for mode in Q.VISUALIZATION_MODES:
        rec.load_state(rows, merges)
        outs = Q.visualization_outputs(rec, n, Q.visualization_params(mode, last, n))
        out[f"visualization/{mode}"] = dict({k: digest(v) for k, v in outs.items()}, inputs=digest(rows))
    rec.close()
    Path(out_path).write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")
    print("wrote", out_path, "runs:", runs, "mean", np.mean(runs, axis=0).tolist())


def free_running_run():
    """One free-running pass of the oracle over the envelope test's stream (printed as JSON)."""
    cam, st, pp, ip = Q.free_running_case()
    first, last = st.integrated_range()
    rec = Q.make(cam, 5_000_000, _lib.load_reference_oracle())
    s = rec.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp, ip,
                       first, last)
    print(json.dumps({"inputs": digest(st.depth.cpu().numpy()), "totals": Q.stream_totals(s)}))
    rec.close()


if __name__ == "__main__":
    if sys.argv[1:] == ["--free-running-run"]:
        free_running_run()
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else str(Path(__file__).resolve().parent / "oracle_answers.json"))
