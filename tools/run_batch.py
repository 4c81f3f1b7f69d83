#!/usr/bin/env python
"""A few batched steps of the bench workload with plain launches (no CUDA graphs), for `ncu` launch lists:
  ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/l.csv python tools/run_batch.py
  python tools/run_batch.py [units] [steps] [features] [--mono-rotation]
--mono-rotation: every unit runs trackingFrame2Frame(mono_rotation = true) (vo_batch_mono_rotation); the essential-matrix
inliers are printed after the PnP inliers.
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from visual_odom_b200 import synth
from visual_odom_b200.capi import Context

mono = "--mono-rotation" in sys.argv[1:]
argv = [a for a in sys.argv[1:] if a != "--mono-rotation"]
units = int(argv[0]) if len(argv) > 0 else 8
steps = int(argv[1]) if len(argv) > 1 else 2
feats = int(argv[2]) if len(argv) > 2 else 2000
us = [synth.stereo_unit(1241, 376, s) for s in range(units)]
ctx = Context(0, max_features=max(2048, feats), max_units=units)
ctx.set_option("graphs", 0)
ctx.batch_configure(1241, 376, units, us[0]["P_l"], us[0]["P_r"])
if mono:
    ctx.batch_mono_rotation(0, [1] * units)
arr, keep, pitch = ctx.make_units([dict(l0=u["l0"], r0=u["r0"], l1=u["l1"], r1=u["r1"], n_select=feats, t_prev=(0.0, 0.0, -0.8)) for u in us])
for _ in range(steps):
    res = ctx.frame_batch(arr, pitch)
print([r["n_inliers"] for r in res])
if mono:
    print([ctx.batch_fetch_mono(u, res[u])["mono"]["n_inliers"] for u in range(units)])
ctx.close()
