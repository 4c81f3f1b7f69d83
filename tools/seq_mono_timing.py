#!/usr/bin/env python
"""Cost of trackingFrame2Frame's mono_rotation branch in the streaming sequence mode, measured on the GPU.

    python tools/seq_mono_timing.py [--frames 40] [--rounds 5] [--json out.json]

On the synthetic 1241x376 drive (synth.stereo_unit, the motion of tests/test_gpu_seq.py) one context runs the same frames
with the option "mono_rotation" off and on, alternated round by round, and reports per mode:
  - pipelined frames/s: vo_seq_submit / vo_seq_wait with two frames in flight
  - one-push latency: median wall time of a synchronous vo_seq_push (submit + wait)
  - kernel launches per frame (vo_kernel_launches)
The card's name and power limit are printed with the numbers; they are part of them."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

STEP_R = np.array([0.001, -0.004, 0.0005])
STEP_T = np.array([0.01, -0.003, -0.2])


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown (nvidia-smi unavailable)"


def frames(w, h, n, seed=31):
    from visual_odom_b200 import synth
    base = synth.stereo_unit(w, h, seed)
    out = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=STEP_R * k, tvec=STEP_T * k)
        out.append((u["l1"], u["r1"]))
    return base, out


def run_pipelined(ctx, base, fr, mono):
    ctx.seq_begin(fr[0][0], fr[0][1], base["P_l"], base["P_r"])
    l0 = ctx.kernel_launches()
    t0 = time.perf_counter()
    ctx.seq_submit(*fr[1])
    for k in range(1, len(fr)):
        if k + 1 < len(fr):
            ctx.seq_submit(*fr[k + 1])
        ctx.seq_wait(want_points=False, mono=mono)
    dt = time.perf_counter() - t0
    return (len(fr) - 1) / dt, (ctx.kernel_launches() - l0) / (len(fr) - 1)


def run_latency(ctx, base, fr, mono):
    ctx.seq_begin(fr[0][0], fr[0][1], base["P_l"], base["P_r"])
    lat = []
    for l, r in fr[1:]:
        t0 = time.perf_counter()
        ctx.seq_push(l, r, want_points=False, mono=mono)
        lat.append(time.perf_counter() - t0)
    return float(np.median(lat))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", help="also write the result here")
    a = ap.parse_args()
    from visual_odom_b200 import capi
    base, fr = frames(1241, 376, a.frames + 1)
    ctx = capi.Context(0, max_features=4096, max_units=2)
    res = {m: dict(fps=[], lat=[], launches=[]) for m in (0, 1)}
    for mono in (0, 1):                               # warm-up: captures both modes' graphs once
        ctx.set_option("mono_rotation", mono)
        run_pipelined(ctx, base, fr[:4], bool(mono))
    for _ in range(a.rounds):
        for mono in (0, 1):
            ctx.set_option("mono_rotation", mono)
            run_pipelined(ctx, base, fr[:3], bool(mono))         # re-capture after the option change, untimed
            fps, launches = run_pipelined(ctx, base, fr, bool(mono))
            res[mono]["fps"].append(fps); res[mono]["launches"].append(launches)
            res[mono]["lat"].append(run_latency(ctx, base, fr, bool(mono)))
    ctx.close()
    out = dict(card=card(), image="1241x376", frames=a.frames, rounds=a.rounds)
    for mono, name in ((0, "off"), (1, "on")):
        r = res[mono]
        out[name] = dict(pipelined_fps=float(np.median(r["fps"])), pipelined_fps_min=float(np.min(r["fps"])),
                         pipelined_fps_max=float(np.max(r["fps"])), push_latency_ms=1e3 * float(np.median(r["lat"])),
                         launches_per_frame=float(np.median(r["launches"])))
    print(f"card (name, power limit): {out['card']}")
    for name in ("off", "on"):
        o = out[name]
        print(f"mono_rotation {name:3s}: pipelined {o['pipelined_fps']:.0f} frames/s "
              f"[{o['pipelined_fps_min']:.0f}, {o['pipelined_fps_max']:.0f}], one-push latency {o['push_latency_ms']:.3f} ms, "
              f"{o['launches_per_frame']:.1f} launches / frame")
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
