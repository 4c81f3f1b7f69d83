#!/usr/bin/env python
"""Cost of the LK window (vo_params.lk_win), measured on the GPU.

    python tools/lk_win_timing.py [--steps 20] [--frames 40] [--json out.json]

- The LK ring's time per launch from vo_lk_kernel_time (CUDA events around the launch; plain launches, graphs 0) on the
  benchmark's workload: 8 units x 2000 features of 1241x376 (synth.stereo_unit), vo_batch_run repeated `steps` times, at
  W = 7, 11, 15, 21, 25, 31 and 32.  W = 21 runs k_lk_ring (lk_ring.cu), every other window k_lk_win (lk_win.cu).
- Sequence-mode frames/s (vo_seq_submit / vo_seq_wait, two frames in flight) on the synthetic 1241x376 drive of
  tests/test_gpu_seq.py at W = 15, 21 and 31, the windows alternated round by round.
The card's name and power limit are read in the same run and printed with the numbers; they are part of them."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

RING_WINDOWS = (7, 11, 15, 21, 25, 31, 32)
SEQ_WINDOWS = (15, 21, 31)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown (nvidia-smi unavailable)"


def ring_ms(units, win, steps):
    from visual_odom_b200.capi import Context
    ctx = Context(0, lk_win=win, max_features=2048, max_units=len(units))
    try:
        ctx.set_option("graphs", 0)
        ctx.batch_configure(1241, 376, len(units), units[0]["P_l"], units[0]["P_r"])
        arr, keep, pitch = ctx.make_units([dict(u, n_select=2000, t_prev=(0.0, 0.0, -0.8)) for u in units])
        ctx.batch_upload(arr, pitch)
        for _ in range(3):
            ctx.batch_run()
        ctx.sync()
        ctx.lk_kernel_time(reset=True)
        for _ in range(steps):
            ctx.batch_run()
        ms, n = ctx.lk_kernel_time(reset=True)
        res = ctx.batch_download(len(units))
        return ms / max(n, 1), n, sum(r["n_valid"] for r in res)
    finally:
        ctx.close()


def seq_fps(ctx, base, fr):
    ctx.seq_begin(fr[0][0], fr[0][1], base["P_l"], base["P_r"])
    t0 = time.perf_counter()
    ctx.seq_submit(*fr[1])
    for k in range(1, len(fr)):
        if k + 1 < len(fr):
            ctx.seq_submit(*fr[k + 1])
        ctx.seq_wait(want_points=False)
    return (len(fr) - 1) / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=20, help="timed vo_batch_run calls per window")
    ap.add_argument("--frames", type=int, default=40, help="frames of the sequence-mode drive")
    ap.add_argument("--rounds", type=int, default=3, help="alternated sequence-mode rounds per window")
    ap.add_argument("--json", help="also write the numbers here")
    a = ap.parse_args()
    from visual_odom_b200 import synth
    from visual_odom_b200.capi import Context
    out = dict(card=card())
    print(f"card: {out['card']}")
    units = [synth.stereo_unit(1241, 376, s) for s in range(8)]
    out["ring"] = {}
    for win in RING_WINDOWS:
        ms, n, valid = ring_ms(units, win, a.steps)
        out["ring"][win] = dict(ms=ms, launches=n, n_valid=valid)
        print(f"LK ring W={win:2d}: {ms:.3f} ms per launch ({n} launches, 8 x 2000 features, 1241x376), {valid} valid matches")
    base = synth.stereo_unit(1241, 376, 31)
    fr = [(base["l0"], base["r0"])]
    for k in range(1, a.frames):
        u = synth.stereo_unit(1241, 376, 31, rvec=synth.SEQ_STEP_R * k, tvec=synth.SEQ_STEP_T * k)
        fr.append((u["l1"], u["r1"]))
    ctxs = {win: Context(0, lk_win=win, max_features=8192) for win in SEQ_WINDOWS}
    fps = {win: [] for win in SEQ_WINDOWS}
    try:
        for win in SEQ_WINDOWS:
            seq_fps(ctxs[win], base, fr[:4])                   # warm-up: allocation, graph capture
        for _ in range(a.rounds):
            for win in SEQ_WINDOWS:
                fps[win].append(seq_fps(ctxs[win], base, fr))
    finally:
        for c in ctxs.values():
            c.close()
    out["seq_fps"] = {win: max(v) for win, v in fps.items()}
    for win in SEQ_WINDOWS:
        print(f"sequence mode W={win:2d}: {max(fps[win]):.0f} frames/s (best of {a.rounds}: "
              + ", ".join(f"{v:.0f}" for v in fps[win]) + f"), 1241x376, {a.frames - 1} frames")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
