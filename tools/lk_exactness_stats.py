#!/usr/bin/env python
"""Kernel-design bookkeeping on the CPU (no GPU): how often could an LK iteration of the benchmark scene take the exact
integer path of k_lk_ring?  Uses the instrumentation hook of the oracle's C restatement (oracle/lk_ref.c, lk_chain_stats):
  former    sum |addend| <= 2^24 on every chain             (the kernel's test before the sign split)
  strips    sum over the kernel's strips of max |running strip sum| <= 2^24
  sign      max(P, N) <= 2^24 on every chain, P and N the sums of the positive products and of |negative products|
            (sum |product| + |total| <= 2^25: the vote the kernel runs)
  truth     every chain prefix and every addend <= 2^24      (the best any test could do)
and how many iterations the sign split accepts although a prefix or an addend leaves +-2^24 (0 if the vote is sound).
This script only reads the oracle; it is not part of any timed or shipped path (DESIGN.md K2 quotes its output)."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import cref, ref_path          # noqa: E402
from visual_odom_b200 import synth         # noqa: E402


def main():
    n_feat = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    seeds = [int(s) for s in sys.argv[2:]] or [0, 1]
    lib = cref.lib()
    lib.lk_stats_enable.argtypes = [C.c_int]
    lib.lk_stats_get.argtypes = [C.c_void_p]
    tot = np.zeros(8, np.int64)
    for s in seeds:
        u = synth.stereo_unit(1241, 376, s, cal=synth.KITTI00)
        corners, _ = cref.fast_detect(u["l0"])
        pts = synth.select_features(corners, n_feat)
        fs = ref_path.FeatureSet(); fs.points = pts.copy(); fs.ages = np.zeros(len(pts), np.int32)
        lib.lk_stats_enable(1)
        ref_path.circular_matching(u["l0"], u["r0"], u["l1"], u["r1"], pts, fs, backend="c")
        out = np.zeros(8, np.int64)
        lib.lk_stats_get(out.ctypes.data_as(C.c_void_p))
        lib.lk_stats_enable(0)
        tot += out
    it = max(int(tot[0]), 1)
    print(f"{len(seeds)} unit(s) x {n_feat} features: {it} Newton iterations over the four calls of the ring")
    for name, k in (("former test (sum |addend|)", 1), ("strip bound", 2), ("sign split (the kernel's vote)", 4),
                    ("truth (prefix sums)", 3)):
        print(f"  exact by {name:30s}: {100.0 * tot[k] / it:5.1f} %")
    print(f"  sign split accepts, a prefix rounds: {int(tot[5])}")


if __name__ == "__main__":
    main()
