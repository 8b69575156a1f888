"""Offline look at how the reference's association race resolves (input: the supporter-set dump of
tools/race_stats.py, <out>_sets.npz): for pairs of supporters of one pixel, who wins as a function of where the two
threads sit in the reference's launch (wave = 2 blocks per SM x SMs x 1024 threads, block, warp, lane;
the SM count is the second argument, 132 = H100 SXM by default)."""
import sys
from collections import defaultdict

import numpy as np

W = 2 * (int(sys.argv[2]) if len(sys.argv) > 2 else 132) * 1024


def main():
    d = np.load(sys.argv[1])
    n, winner, slots, sec = d["n"], d["winner"], d["slots"], d["secondary"]
    print("records", len(n), "set sizes", np.bincount(n)[:8])
    two = n == 2
    a, b = slots[two, 0].astype(np.int64), slots[two, 1].astype(np.int64)   # a < b
    low_wins = winner[two] == 0
    sa, sb = (sec[two] & 1).astype(bool), ((sec[two] >> 1) & 1).astype(bool)
    wave_a, wave_b = a // W, b // W
    both_primary = ~sa & ~sb
    print("pairs", two.sum(), "both primary", both_primary.sum())

    def report(name, mask):
        if mask.sum() == 0:
            return
        print(f"  {name:44s} n={mask.sum():7d}  lower slot wins {low_wins[mask].mean():.3f}")

    for kind, km in (("primary/primary", both_primary), ("secondary/secondary", sa & sb)):
        print(kind)
        same_wave = km & (wave_a == wave_b)
        report("different wave", km & (wave_a != wave_b))
        report("same wave", same_wave)
        ra, rb = a % W, b % W
        blk_a, blk_b = ra // 1024, rb // 1024
        same_block = same_wave & (blk_a == blk_b)
        report("same block", same_block)
        warp_a, warp_b = (ra % 1024) // 32, (rb % 1024) // 32
        report("same block, same warp", same_block & (warp_a == warp_b))
        for lo, hi in ((1, 1), (2, 3), (4, 7), (8, 15), (16, 31)):
            dw = warp_b - warp_a
            report(f"same block, warp distance {lo}-{hi}", same_block & (dw >= lo) & (dw <= hi))
        diff_block = same_wave & (blk_a != blk_b)
        report("different block", diff_block)
        db = blk_b - blk_a
        sms = W // 2048
        for lo, hi in ((1, 1), (2, 7), (8, 31), (32, sms - 1), (sms, sms), (sms + 1, 2 * sms - 1)):
            report(f"block distance {lo}-{hi}", diff_block & (db >= lo) & (db <= hi))
        report(f"different block, same SM parity (d % {sms} == 0)", diff_block & (db % sms == 0))
        # does the position inside the block matter across blocks?
        for name, m in (("a earlier in its block than b", (ra % 1024) < (rb % 1024)), ("a later in its block than b", (ra % 1024) > (rb % 1024))):
            report("different block, " + name, diff_block & m)
        pos_diff = (rb % 1024) - (ra % 1024)
        for lo, hi in ((-1023, -512), (-511, -128), (-127, -1), (0, 127), (128, 511), (512, 1023)):
            report(f"different block, in-block offset b-a in [{lo},{hi}]", diff_block & (pos_diff >= lo) & (pos_diff <= hi))
    print("mixed kinds (one primary, one secondary), same wave")
    mixed = (sa != sb) & (wave_a == wave_b)
    prim_wins = np.where(sa, ~low_wins, low_wins)
    print(f"  n={mixed.sum()} primary wins {prim_wins[mixed].mean():.3f}; when primary is the lower slot {prim_wins[mixed & ~sa].mean():.3f}, "
          f"when it is the higher slot {prim_wins[mixed & sa].mean():.3f}")
    ra, rb = a % W, b % W
    same_block = mixed & (ra // 1024 == rb // 1024)
    print(f"  same block n={same_block.sum()} primary wins {prim_wins[same_block].mean():.3f}")


if __name__ == "__main__":
    main()
