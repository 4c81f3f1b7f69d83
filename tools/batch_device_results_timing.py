#!/usr/bin/env python
"""Host waits against device waits of the batched mode, measured on the GPU.

    python tools/batch_device_results_timing.py [--seconds 4] [--rounds 3] [--json out.json] [--check]

The bench workload (1241x376 synthetic KITTI units, 8 units x 2000 selected features per submission, three submissions
in flight on disjoint slot ranges, images from device memory through vo_batch_submit_device) is retired three ways:

  host+lists    vo_batch_wait + "batch_outputs" = 1 + vo_batch_outputs of every unit (bench.py's e2e retirement)
  host          vo_batch_wait of the records only ("batch_outputs" = 0)
  device        vo_batch_wait_device of the records and every list (pts4, kept_idx, points3D, inliers) into CUDA tensors
                reused every step ("batch_outputs" = 0), then a trivial torch consumer on the same stream (the sum of the
                n_valid counts, accumulated on the device); the final synchronise is inside the timed window

The three modes alternate round by round (the order reversed every other round); each round runs for --seconds, and the
median over the rounds is reported: frames/s, host time per step spent inside the library calls (submit + wait, and the
vo_batch_outputs reads), kernel launches per submission and per wait.  The card's name, power limit and max SM clock are
read in the same call and printed with the numbers; they are part of them.

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
PTS_CAP = 2048
MODES = ("host+lists", "host", "device")


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
                inputs="device (vo_batch_submit_device)", pts_cap=PTS_CAP, modes=list(MODES), rounds=a.rounds, seconds=a.seconds)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown (nvidia-smi unavailable)"


def run_mode(ctx, dev, mode, seconds, outs, acc):
    """Pipelined submissions for `seconds`: (frames/s, host ms per step inside the calls, launches per submission,
    launches per wait)."""
    import torch
    ctx.set_option("batch_outputs", 1 if mode == "host+lists" else 0)
    host_s = [0.0]
    launches = {"submit": 0, "wait": 0}

    def timed(kind, fn, *args, **kw):
        l0, t0 = ctx.kernel_launches(), time.perf_counter()
        r = fn(*args, **kw)
        host_s[0] += time.perf_counter() - t0
        launches[kind] += ctx.kernel_launches() - l0
        return r

    def submit(slot):
        timed("submit", ctx.batch_submit_device, dev, slot * B)

    def wait(slot):
        if mode == "device":
            out = timed("wait", ctx.batch_wait_device, slot * B, B, out=outs[slot])
            acc.add_(out["counts"][:, 3].sum())              # the consumer: stream-ordered, no host wait
            return
        res = timed("wait", ctx.batch_wait, slot * B, B)
        if mode == "host+lists":
            for u in range(B):
                timed("wait", ctx.batch_outputs, slot * B + u, res[u])

    for k in range(DEPTH - 1):                  # warm-up: every slot range once
        submit(k)
    for s in range(2 * DEPTH):
        submit((s + DEPTH - 1) % DEPTH)
        wait(s % DEPTH)
    for s in range(2 * DEPTH, 3 * DEPTH - 1):
        wait(s % DEPTH)
    torch.cuda.synchronize()
    for k in range(DEPTH - 1):
        submit(k)
    host_s[0] = 0.0
    launches.update(submit=0, wait=0)
    t0, s = time.perf_counter(), 0
    while True:
        submit((s + DEPTH - 1) % DEPTH)
        wait(s % DEPTH)
        s += 1
        if time.perf_counter() - t0 >= seconds:
            break
    for k in range(s, s + DEPTH - 1):           # drain inside the timed region: every frame counted has finished
        wait(k % DEPTH)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    steps = s + DEPTH - 1                       # waits in the timed region (the DEPTH - 1 first were submitted before it)
    return steps * B / dt, 1e3 * host_s[0] / steps, launches["submit"] / s, launches["wait"] / steps


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
    ctx = Context(0, max_features=2048, max_units=DEPTH * B)
    ctx.batch_configure(W, H, DEPTH * B, us[0]["P_l"], us[0]["P_r"])
    dev = [dict({k: torch.from_numpy(u[k]).cuda() for k in ("l0", "r0", "l1", "r1")}, n_select=FEATS, t_prev=T_PREV) for u in us]
    outs = [ctx.batch_dresults_alloc(B, pts_cap=PTS_CAP) for _ in range(DEPTH)]
    acc = torch.zeros((), dtype=torch.int64, device="cuda")
    res = {m: [] for m in MODES}
    for r in range(a.rounds):
        for m in (MODES if r % 2 == 0 else MODES[::-1]):
            res[m].append(run_mode(ctx, dev, m, a.seconds, outs, acc))
    ctx.close()
    med = lambda m, i: float(np.median([x[i] for x in res[m]]))
    out = dict(card=gpu, plan=plan(a), results=[
        dict(mode=m, frames_per_s=med(m, 0), host_ms_per_step=med(m, 1), launches_per_submission=med(m, 2),
             launches_per_wait=med(m, 3), rounds=[round(x[0], 1) for x in res[m]]) for m in MODES])
    print(f"card: {gpu}")
    print(f"{'mode':>11} {'frames/s':>10} {'host ms/step':>13} {'launches/sub':>13} {'launches/wait':>14}  rounds")
    for e in out["results"]:
        print(f"{e['mode']:>11} {e['frames_per_s']:>10.1f} {e['host_ms_per_step']:>13.3f} {e['launches_per_submission']:>13.1f} "
              f"{e['launches_per_wait']:>14.2f}  {e['rounds']}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
