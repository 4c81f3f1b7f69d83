#!/usr/bin/env python
"""Cost of trackingFrame2Frame's mono_rotation branch in the batched mode, measured on the GPU.

    python tools/batch_mono_timing.py [--seconds 4] [--rounds 3] [--json out.json] [--check]

The bench workload (1241x376 synthetic KITTI units, 8 units x 2000 selected features per submission, three submissions
in flight on disjoint slot ranges, as bench.py's e2e loop, with "batch_outputs" = 1 and every unit's lists read) runs with
0, 1 and all 8 units of each submission switched on (vo_batch_mono_rotation), from pinned host images (vo_batch_submit)
and from images in device memory (vo_batch_submit_device).  The six modes alternate round by round; each round runs for
--seconds, and the median frames/s over the rounds is reported with the kernel launches per submission.  The card's name,
power limit and max SM clock are read in the same call and printed with the numbers; they are part of them.

--check validates the arguments and prints the plan without touching a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H, B, FEATS, DEPTH = 1241, 376, 8, 2000, 3
T_PREV = (0.0, 0.0, -0.8)
ON_COUNTS = (0, 1, 8)
INPUTS = ("host", "device")


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--seconds", type=float, default=4.0, help="length of one round of one mode")
    ap.add_argument("--rounds", type=int, default=3, help="rounds per mode (at least 3; the median is reported)")
    ap.add_argument("--json", help="also write the results here")
    ap.add_argument("--check", action="store_true", help="validate the arguments, print the plan, run nothing")
    a = ap.parse_args(argv)
    if a.rounds < 3:
        ap.error("--rounds must be at least 3")
    if not a.seconds > 0:
        ap.error("--seconds must be positive")
    return a


def plan(a):
    return dict(size=[W, H], units_per_submission=B, features=FEATS, in_flight=DEPTH, units_configured=DEPTH * B,
                modes=[dict(inputs=i, units_on=n) for i in INPUTS for n in ON_COUNTS], rounds=a.rounds, seconds=a.seconds)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown (nvidia-smi unavailable)"


def pattern(n_on):
    """The switch of each of the DEPTH * B configured units: the first n_on units of every submission's range on."""
    return [1 if (u % B) < n_on else 0 for u in range(DEPTH * B)]


def run_mode(ctx, host, dev, pitch, inputs, n_on, seconds):
    """Pipelined submissions for `seconds`: (frames/s, launches per submission)."""
    ctx.batch_mono_rotation(0, pattern(n_on))

    def submit(slot):
        if inputs == "host":
            ctx.batch_submit(host, slot * B, pitch)
        else:
            ctx.batch_submit_device(dev, slot * B)

    def wait(slot):
        if n_on:
            res, _ = ctx.batch_wait_mono(slot * B, B)
        else:
            res = ctx.batch_wait(slot * B, B)
        for u in range(B):
            ctx.batch_outputs(slot * B + u, res[u])

    for k in range(DEPTH - 1):                  # warm-up: every slot range once
        submit(k)
    for s in range(2 * DEPTH):
        submit((s + DEPTH - 1) % DEPTH)
        wait(s % DEPTH)
    for s in range(2 * DEPTH, 3 * DEPTH - 1):
        wait(s % DEPTH)
    for k in range(DEPTH - 1):
        submit(k)
    l0, t0, s = ctx.kernel_launches(), time.perf_counter(), 0
    while True:
        submit((s + DEPTH - 1) % DEPTH)
        wait(s % DEPTH)
        s += 1
        if time.perf_counter() - t0 >= seconds:
            break
    for k in range(s, s + DEPTH - 1):           # drain inside the timed region: every frame counted has finished
        wait(k % DEPTH)
    dt = time.perf_counter() - t0
    return (s + DEPTH - 1) * B / dt, (ctx.kernel_launches() - l0) / s      # the DEPTH - 1 first were launched before l0


def main(argv=None):
    a = parse(argv)
    if a.check:
        print(json.dumps(dict(plan=plan(a)), indent=1))
        return 0
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        print("no CUDA device: nothing measured", file=sys.stderr)
        return 1
    from visual_odom_b200 import synth
    from visual_odom_b200.capi import Context
    gpu = card()
    us = [synth.stereo_unit(W, H, s) for s in range(B)]
    pinned = [{k: torch.from_numpy(u[k]).pin_memory() for k in ("l0", "r0", "l1", "r1")} for u in us]
    ctx = Context(0, max_features=2048, max_units=DEPTH * B)
    ctx.set_option("batch_outputs", 1)
    ctx.batch_configure(W, H, DEPTH * B, us[0]["P_l"], us[0]["P_r"])
    host, keep, pitch = ctx.make_units([dict({k: p[k].numpy() for k in p}, n_select=FEATS, t_prev=T_PREV) for p in pinned])
    dev = [dict({k: torch.from_numpy(u[k]).cuda() for k in ("l0", "r0", "l1", "r1")}, n_select=FEATS, t_prev=T_PREV) for u in us]
    modes = [(i, n) for i in INPUTS for n in ON_COUNTS]
    rates = {m: [] for m in modes}
    launches = {}
    for r in range(a.rounds):
        for m in (modes if r % 2 == 0 else modes[::-1]):
            fps, lps = run_mode(ctx, host, dev, pitch, m[0], m[1], a.seconds)
            rates[m].append(fps)
            launches[m] = lps
    ctx.close()
    out = dict(card=gpu, plan=plan(a), results=[
        dict(inputs=i, units_on=n, frames_per_s=float(np.median(rates[(i, n)])), rounds=[round(x, 1) for x in rates[(i, n)]],
             launches_per_submission=launches[(i, n)]) for (i, n) in modes])
    print(f"card: {gpu}")
    print(f"{'inputs':>7} {'units on':>9} {'frames/s':>10} {'launches/sub':>13}  rounds")
    for e in out["results"]:
        print(f"{e['inputs']:>7} {e['units_on']:>9} {e['frames_per_s']:>10.1f} {e['launches_per_submission']:>13.1f}  {e['rounds']}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
