#!/usr/bin/env python
"""A/B of the LK ring kernel's instantiations / work-item sizes on the bench workload (one GPU, single stream, plain launches):
  LK_KERNELS=4:8:2,4:12:2 python tools/lk_ab.py [units] [features] [steps]      (4:<CTAs per SM>:<phases per work item>)
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
kernels = os.environ.get("LK_KERNELS", "4:8:2,4:8:16,4:8:1,4:8:4,4:10:2,4:12:2").split(",")      # 4:ctas_per_sm:span (span 16 = one item per feature-ring)
unit_sets = [[synth.stereo_unit(1241, 376, s0 + s) for s in range(units)] for s0 in (0, 1000)]
out = {}
got = {}
for k in kernels:
    kk = k.split(":")
    ctx = Context(0, max_features=max(2048, feats), max_units=units)
    ctx.set_option("graphs", 0)
    ctx.set_option("batch_streams", 1)
    ctx.set_option("lk_ctas_per_sm", int(kk[1]) if len(kk) > 1 else 0)
    ctx.set_option("lk_span", int(kk[2]) if len(kk) > 2 else 0)
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
            out[f"lk_v{k}_ms"] = ms / max(n, 1)
        res = ctx.batch_download(units)
        got[k] += [ctx.batch_fetch(u, res[u]) for u in range(units)]
        if j == 0:
            out[f"lk_v{k}_inliers"] = [r["n_inliers"] for r in res]
    ctx.close()
a = got[kernels[0]]
for k in kernels[1:]:
    b = got[k]
    out[f"identical_{kernels[0]}_{k}"] = bool(all(np.array_equal(x[key], y[key]) for x, y in zip(a, b)
                                                  for key in ("l0", "r0", "l1", "r1", "kept_idx", "inliers")))
print(json.dumps(out))
