#!/usr/bin/env python
"""Developer probe (run on a GPU): how does the reference's supporting-surfel race
(atomicCAS, kernels.cu:1688) actually resolve, and which reproducible tie-break of the product
lands inside the reference's own run-to-run envelope?

1. Teacher-forced samples: oracle A runs the stream frame by frame; at sampled frames the state
   before the frame is copied into oracle B and into the product (one load per tie-break
   variant), everybody integrates the same frame, and the merge counts are compared. The
   supporter SETS of the frame come from oracle/cpu_walk (independent of the product), the winner
   from oracle A's raster: who wins as a function of primary/secondary, slot index, launch wave.
2. Free-running totals over the whole stream for every variant and for three oracle runs.

Writes probe_out/race_stats.json."""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import cpu_walk  # noqa: E402
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402

INV = 0xFFFFFFFF
REF_WAVE = None  # the reference's AssociateSurfels launch wave: 2 resident 1024-thread blocks per SM x SMs (set in main)


def u16(h, w):
    return torch.zeros((h, w), dtype=torch.uint16, device="cuda")


def collect_sets(ev_pixel, ev_key, sup, cnt, frame, store, max_set=6):
    """Contested pixels of one frame as fixed-width records for an offline fit of the arrival order:
    frame, pixel, set size, winner position, slots (padded with 0xFFFFFFFF), secondary bits."""
    order = np.lexsort((ev_key & 0x7FFFFFFF, ev_pixel))
    px, key = ev_pixel[order], ev_key[order]
    bounds = np.flatnonzero(np.diff(px)) + 1
    starts = np.concatenate([[0], bounds])
    ends = np.concatenate([bounds, [len(px)]])
    sup = sup.reshape(-1)
    cnt = cnt.reshape(-1)
    for s, e in zip(starts, ends):
        n = e - s
        if n < 2 or n > max_set or cnt[px[s]] != n:
            continue
        idx = key[s:e] & 0x7FFFFFFF
        hit = np.flatnonzero(idx == sup[px[s]])
        if len(hit) == 0:
            continue
        rec = np.full(max_set, 0xFFFFFFFF, np.uint32)
        rec[:n] = idx
        store["frame"].append(frame)
        store["pixel"].append(int(px[s]))
        store["n"].append(n)
        store["winner"].append(int(hit[0]))
        store["slots"].append(rec)
        store["secondary"].append(int(sum(((int(key[s + k]) >> 31) & 1) << k for k in range(n))))


def winner_stats(ev_pixel, ev_key, sup, cnt, acc):
    """Accumulates, over the multi-supporter pixels whose CPU supporter set has the size the GPU
    counted, who won the reference's race."""
    order = np.argsort(ev_pixel, kind="stable")
    px, key = ev_pixel[order], ev_key[order]
    bounds = np.flatnonzero(np.diff(px)) + 1
    starts = np.concatenate([[0], bounds])
    ends = np.concatenate([bounds, [len(px)]])
    sup = sup.reshape(-1)
    cnt = cnt.reshape(-1)
    for s, e in zip(starts, ends):
        n = e - s
        if n < 2:
            continue
        p = px[s]
        if cnt[p] != n:
            acc["set_size_mismatch"] += 1
            continue
        keys = key[s:e]
        idx = keys & 0x7FFFFFFF
        sec = (keys >> 31).astype(bool)
        w = sup[p]
        hit = np.flatnonzero(idx == w)
        acc["multi_pixels"] += 1
        if len(hit) == 0:
            acc["winner_not_in_set"] += 1
            continue
        wi = hit[0]
        has_p, has_s = (~sec).any(), sec.any()
        if has_p and has_s:
            acc["mixed"] += 1
            acc["mixed_secondary_wins"] += int(sec[wi])
            k = f"mixed_p{min(int((~sec).sum()), 3)}_s{min(int(sec.sum()), 3)}"
            acc[k] = acc.get(k, 0) + 1
            acc[k + "_secwins"] = acc.get(k + "_secwins", 0) + int(sec[wi])
            # same launch wave only
            waves = idx // REF_WAVE
            if (waves == waves[0]).all():
                acc["mixed_samewave"] += 1
                acc["mixed_samewave_secondary_wins"] += int(sec[wi])
        same_kind = not (has_p and has_s)
        if same_kind and n == 2:
            acc["pair_same_kind"] += 1
            acc["pair_same_kind_lower_index_wins"] += int(idx[wi] == idx.min())
            waves = idx // REF_WAVE
            if waves[0] != waves[1]:
                acc["pair_two_waves"] += 1
                acc["pair_two_waves_lower_wave_wins"] += int(waves[wi] == waves.min())
            else:
                acc["pair_one_wave"] += 1
                acc["pair_one_wave_lower_index_wins"] += int(idx[wi] == idx.min())
                # distance in blocks of 1024 slots
                far = abs(int(idx[0]) - int(idx[1])) >= 32 * 1024
                acc["pair_one_wave_far" if far else "pair_one_wave_near"] += 1
                acc["pair_one_wave_far_lower_wins" if far else "pair_one_wave_near_lower_wins"] += int(idx[wi] == idx.min())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=500)
    ap.add_argument("--sample-every", type=int, default=16)
    ap.add_argument("--cap", type=int, default=5_000_000)
    ap.add_argument("--free-runs", type=int, default=2)
    ap.add_argument("--out", default="probe_out/race_stats.json")
    args = ap.parse_args()

    global REF_WAVE
    REF_WAVE = 2 * torch.cuda.get_device_properties(0).multi_processor_count * 1024
    prod = _lib.load_product()
    ref = _lib.load_reference_oracle()
    cam = S.Camera.tum(640, 480)
    W, H = cam.width, cam.height
    t0 = time.time()
    st = S.make_stream(cam, args.frames, device="cuda")
    print(f"stream: {args.frames} frames in {time.time() - t0:.1f}s", flush=True)
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    first, last = st.integrated_range()
    K = pp.outlier_filtering_frame_count

    # (name, wave W, early fraction q of the secondaries, fraction b of the pixels in slot order, lanes that keep
    #  their order inside the shuffled order)
    # name -> knobs (sm_configure "tiebreak_*"): wave W, early fraction q of the secondaries and fraction b of the pixels in
    # slot order for the first wave / for the later waves (q1, b1; absent = same), lanes that keep their order
    def rule(wave=REF_WAVE, q=0.01, b=0.25, lanes=32, phase=0, q1=-1.0, b1=-1.0):
        return {"wave": wave, "early_fraction": q, "index_order_fraction": b, "lanes": lanes, "wave_offset": phase,
                "early_fraction_later": q1, "index_order_fraction_later": b1}
    variants = [("plain", rule(wave=0, q=0, b=0, lanes=1)), ("wave_q0.01_b0.25", rule()), ("wave_q0.02_b0.25", rule(q=0.02))]
    for q1, b1 in ((0.03, -1.0), (0.04, -1.0), (0.06, -1.0), (0.03, 0.45), (0.04, 0.45), (0.06, 0.45), (0.04, 0.7), (0.08, 0.7)):
        variants.append((f"wave_q0.01_b0.25_later_q{q1}_b{b1 if b1 >= 0 else 'same'}", rule(q1=q1, b1=b1)))

    def set_variant(rec, knobs):
        for key in ("wave_offset", "lanes", "wave", "early_fraction", "index_order_fraction", "early_fraction_later",
                    "index_order_fraction_later"):
            rec.configure("tiebreak_" + key, knobs[key])

    def mk(lib=None):
        return R.CUDASurfelReconstruction(args.cap, W, H, cam.fx, cam.fy, cam.cx, cam.cy, lib=lib)

    rec_a, rec_b, rec_p = mk(ref), mk(ref), mk()

    def pre(rec, frame):
        others = [st.depth[frame - (i + 1)] for i in range(K // 2)] + [st.depth[frame + (i + 1)] for i in range(K // 2)]
        d = u16(H, W)
        n = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
        r = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        rec.preprocess(None, pp, st.depth[frame], others, st.others_TR_reference[frame], d, n, r)
        return d, n, r

    acc = {k: 0 for k in ("multi_pixels", "winner_not_in_set", "set_size_mismatch", "mixed", "mixed_secondary_wins",
                          "mixed_samewave", "mixed_samewave_secondary_wins", "pair_same_kind",
                          "pair_same_kind_lower_index_wins", "pair_two_waves", "pair_two_waves_lower_wave_wins",
                          "pair_one_wave", "pair_one_wave_lower_index_wins", "pair_one_wave_far", "pair_one_wave_near",
                          "pair_one_wave_far_lower_wins", "pair_one_wave_near_lower_wins")}
    samples, agree, flagdiff = [], {}, {}
    sets = {k: [] for k in ("frame", "pixel", "n", "winner", "slots", "secondary")}
    t0 = time.time()
    for frame in range(first, last):
        d0, n0, r0 = pre(rec_a, frame)
        sample = (frame - first) % args.sample_every == args.sample_every // 2
        if sample:
            rows, n_before, merges_before = rec_a.dump_state()
            rec_b.load_state(rows, merges_before)
            entry = {"frame": frame, "n_before": int(n_before)}
            winners, flags = {}, {}
            for name, knobs in variants:
                rec_p.load_state(rows, merges_before)
                set_variant(rec_p, knobs)
                rec_p.integrate(None, frame, ip, d0.clone(), n0, r0, st.color[frame], st.global_T_frame[frame],
                                st.frame_T_global[frame])
                entry[name] = int(rec_p.surfels_size() - rec_p.surfel_count()) - int(merges_before)
                winners[name] = rec_p.download_rasters()["supporting_surfels"]
                flags[name] = rec_p.dump_state()[0][7, :n_before] < 0
            rec_b.integrate(None, frame, ip, d0.clone(), n0, r0, st.color[frame], st.global_T_frame[frame],
                            st.frame_T_global[frame])
            entry["oracle_b"] = int(rec_b.surfels_size() - rec_b.surfel_count()) - int(merges_before)
        rec_a.integrate(None, frame, ip, d0.clone(), n0, r0, st.color[frame], st.global_T_frame[frame],
                        st.frame_T_global[frame])
        if sample:
            entry["oracle_a"] = int(rec_a.surfels_size() - rec_a.surfel_count()) - int(merges_before)
            ras = rec_a.download_rasters()
            _, ev_p, ev_k = cpu_walk.associate_events(rows, frame, cam.fx, cam.fy, cam.cx, cam.cy, st.frame_T_global[frame],
                                                      d0.cpu().numpy(), n0.cpu().numpy(), ip.sensor_noise_factor,
                                                      ip.normal_compatibility_threshold_deg, ip.depth_scaling)
            winner_stats(ev_p, ev_k, ras["supporting_surfels"], ras["supporting_surfel_counts"], acc)
            collect_sets(ev_p, ev_k, ras["supporting_surfels"], ras["supporting_surfel_counts"], frame, sets)
            # a second look at the same frame from oracle B: is the winner reproducible from run to run?
            ras_b = rec_b.download_rasters()
            both = (ras["supporting_surfel_counts"] > 1)
            acc["contested_pixels_ab"] = acc.get("contested_pixels_ab", 0) + int(both.sum())
            acc["contested_same_winner_ab"] = acc.get("contested_same_winner_ab", 0) + int(
                (ras["supporting_surfels"][both] == ras_b["supporting_surfels"][both]).sum())
            # the per-frame quantities the envelope tests look at: same winner as oracle A on the contested pixels,
            # merge flags that differ from oracle A's (oracle B gives the reference's own run-to-run figure)
            flags_a = rec_a.dump_state()[0][7, :n_before] < 0
            flags_b = rec_b.dump_state()[0][7, :n_before] < 0
            agree["oracle_b"] = agree.get("oracle_b", 0) + int((ras_b["supporting_surfels"][both] == ras["supporting_surfels"][both]).sum())
            flagdiff["oracle_b"] = flagdiff.get("oracle_b", 0) + int((flags_b != flags_a).sum())
            for name in winners:
                agree[name] = agree.get(name, 0) + int((winners[name][both] == ras["supporting_surfels"][both]).sum())
                flagdiff[name] = flagdiff.get(name, 0) + int((flags[name] != flags_a).sum())
            samples.append(entry)
            print(json.dumps(entry), flush=True)
    print(f"teacher-forced pass: {time.time() - t0:.1f}s")
    sums = {k: sum(e[k] for e in samples) for k in samples[0] if k not in ("frame", "n_before")}
    print("merge-count sums over the samples:", json.dumps(sums, indent=1))
    for lo, hi in ((0, REF_WAVE), (REF_WAVE, 1 << 31)):
        part = [e for e in samples if lo <= e["n_before"] < hi]
        if part:
            print(f"  samples with {lo} <= N < {hi}: " + ", ".join(
                f"{k} {sum(e[k] for e in part) - sum(e['oracle_a'] for e in part):+d}" for k in part[0] if k not in ("frame", "n_before", "oracle_a")))
    print("race statistics:", json.dumps(acc, indent=1))
    print("per-frame agreement with oracle A over the sampled frames (contested pixels: %d):" % acc["contested_pixels_ab"])
    for name in agree:
        print(f"  {name:44s} same winner {agree[name] / max(acc['contested_pixels_ab'], 1):.4f}   differing merge flags {flagdiff[name]:7d}"
              f"  ({flagdiff[name] / max(flagdiff['oracle_b'], 1):.2f} x oracle B)")

    # ---- free-running totals ----
    free = {}
    for rep in range(3):
        rec_a.reset()
        s_ = rec_a.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global, st.others_TR_reference, pp,
                              ip, first, last)
        free[f"oracle_{rep}"] = [int(s_.surfels_size), int(s_.surfel_count)]
    for name, knobs in variants:
        for rep in range(args.free_runs):
            rec_p.reset()
            set_variant(rec_p, knobs)
            s_ = rec_p.stream_run(None, st.depth, st.color, st.global_T_frame, st.frame_T_global,
                                  st.others_TR_reference, pp, ip, first, last)
            free[name if rep == 0 else f"{name}_{rep}"] = [int(s_.surfels_size), int(s_.surfel_count)]
    print("free-running [surfels_size, surfel_count] after the stream:")
    for k, v in free.items():
        print(f"  {k:44s} {v[0]:9d} {v[1]:9d}   merged {v[0] - v[1]:8d}")
    Path(args.out).parent.mkdir(exist_ok=True)
    Path(args.out).write_text(json.dumps({"samples": samples, "sums": sums, "race": acc, "free": free, "same_winner_as_oracle_a": agree,
                                          "differing_merge_flags_vs_oracle_a": flagdiff}, indent=1))
    np.savez_compressed(str(Path(args.out).with_suffix("")) + "_sets.npz", frame=np.array(sets["frame"], np.uint16),
                        pixel=np.array(sets["pixel"], np.uint32), n=np.array(sets["n"], np.uint8),
                        winner=np.array(sets["winner"], np.uint8), slots=np.array(sets["slots"], np.uint32),
                        secondary=np.array(sets["secondary"], np.uint8),
                        n_before=np.array([[e["frame"], e["n_before"]] for e in samples], np.uint32))


if __name__ == "__main__":
    main()
