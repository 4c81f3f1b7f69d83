#!/usr/bin/env python
"""A few frames of the streaming sequence mode with plain launches (no CUDA graphs); tools/launch_summary.py profiles it."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from visual_odom_b200 import synth

W, H = 1241, 376


def stereo_frames(n):
    """The first stereo pair, its projection matrices and n later pairs of a forward-moving synthetic rig."""
    base = synth.stereo_unit(W, H, 31)
    frames = [(base["l0"], base["r0"])]
    for k in range(1, n + 1):
        u = synth.stereo_unit(W, H, 31, rvec=np.array([0.001, -0.004, 0.0005]) * k, tvec=np.array([0.01, -0.003, -0.2]) * k)
        frames.append((u["l1"], u["r1"]))
    return frames, base["P_l"], base["P_r"]


if __name__ == "__main__":
    from visual_odom_b200.capi import Context
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    graphs = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    frames, P_l, P_r = stereo_frames(n)
    ctx = Context(0, max_features=4096, max_units=1)
    ctx.set_option("graphs", graphs)
    ctx.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    for k in range(1, n + 1):
        got = ctx.seq_push(frames[k][0], frames[k][1], want_points=False)
    print(got["n_features"], got["n_valid"], got["n_inliers"])
    ctx.close()
