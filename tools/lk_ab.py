#!/usr/bin/env python
"""A/B of the LK ring kernel's work-item sizes on the bench workload (one GPU, single stream, plain launches):
  LK_SPANS=2,16 python tools/lk_ab.py [units] [features] [steps]      (phases per work item; 16 = one item per feature-ring)
Prints the average CUDA-event time of the LK launch per configuration and checks that all of them produce identical
point lists / inlier lists (bit-exact).  Every configuration runs on a fresh context, on one set of units and then on
another: a configuration that skipped work would be left with the other set's (or the previous context's) outputs.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from visual_odom_b200 import synth
from visual_odom_b200.capi import Context

units = int(sys.argv[1]) if len(sys.argv) > 1 else 8
feats = int(sys.argv[2]) if len(sys.argv) > 2 else 2000
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
spans = os.environ.get("LK_SPANS", "2,16,1,4").split(",")
unit_sets = [[synth.stereo_unit(1241, 376, s0 + s) for s in range(units)] for s0 in (0, 1000)]
out = {}
got = {}
for k in spans:
    ctx = Context(0, max_features=max(2048, feats), max_units=units)
    ctx.set_option("graphs", 0)
    ctx.set_option("batch_streams", 1)
    ctx.set_option("lk_span", int(k))
    ctx.batch_configure(1241, 376, units, unit_sets[0][0]["P_l"], unit_sets[0][0]["P_r"])
    got[k] = []
    for j, us in enumerate(unit_sets):
        arr, keep, pitch = ctx.make_units([dict(l0=u["l0"], r0=u["r0"], l1=u["l1"], r1=u["r1"], n_select=feats, t_prev=(0.0, 0.0, -0.8))
                                           for u in us])
        ctx.batch_upload(arr, pitch)
        ctx.batch_run()
        ctx.sync()
        if j == 0:                 # timing on the first set
            for _ in range(2):
                ctx.batch_run()
            ctx.sync()
            ctx.lk_kernel_time(reset=True)
            for _ in range(steps):
                ctx.batch_run()
            ctx.sync()
            ms, n = ctx.lk_kernel_time(reset=True)
            out[f"lk_span{k}_ms"] = ms / max(n, 1)
        res = ctx.batch_download(units)
        got[k] += [ctx.batch_fetch(u, res[u]) for u in range(units)]
        if j == 0:
            out[f"lk_span{k}_inliers"] = [r["n_inliers"] for r in res]
    ctx.close()
a = got[spans[0]]
for k in spans[1:]:
    b = got[k]
    out[f"identical_{spans[0]}_{k}"] = bool(all(np.array_equal(x[key], y[key]) for x, y in zip(a, b)
                                                for key in ("l0", "r0", "l1", "r1", "kept_idx", "inliers")))
print(json.dumps(out))
