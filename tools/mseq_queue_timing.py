#!/usr/bin/env python
"""A queue of drives of unequal length through the multi-sequence mode, with starts against consecutive batches.

    python tools/mseq_queue_timing.py [--scale 0.01] [--size 640x240] [--slots 2,4,8] [--rounds 3] [--json out.json]
    python tools/mseq_queue_timing.py --check        # the step counts of the full-length queue, no GPU needed

The queue is the KITTI odometry training set's 11 sequence lengths (4541, 1101, 4661, 801, 271, 2761, 1101, 1101, 4071,
1591 and 1201 frames) times --scale (at least 3 frames each), as synthetic drives at --size (synth.stereo_unit; each
drive replays a pool of 8 rendered frames back and forth, with its own motion).  Per slot count N, alternated round by
round on one context:
  - "start":   vo_mseq_open(N) and vo_mseq_submit_start: each drive starts in the first slot that frees, in order
  - "batches": consecutive vo_mseq_begin batches of N drives, each run until its longest drive ends (NULL pairs retire
               the shorter ones)
both with two submissions in flight.  Reported per mode (median over the rounds): aggregate frames/s (sequence-frames per
second of wall time), submissions, mean live slots per submission, the step latency (wall time between consecutive
waits) of submissions with starts and of plain ones, and kernel launches per plain and per start submission.  Then one
idle-slot case: 8 opened slots with 2 live drives against vo_mseq_begin of the same 2 (empty slots still take part in
the pyramid and FAST launches).  The card's name, power limit and max SM clock, read in the same run, are printed with
the numbers; they are part of them."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from run_sequences import queue_schedule

KITTI_LENGTHS = [4541, 1101, 4661, 801, 271, 2761, 1101, 1101, 4071, 1591, 1201]
POOL = 8


def drives(w, h, n):
    from visual_odom_b200 import synth
    out = []
    for d in range(n):
        rng = np.random.default_rng(200 + d)
        r = rng.uniform(-0.003, 0.003, 3) * np.array([1.0, 1.0, 0.25])
        t = np.array([0.0, 0.0, -0.2]) + rng.uniform(-0.02, 0.02, 3)
        base = synth.stereo_unit(w, h, 300 + d)
        fr = [(base["l0"], base["r0"])]
        for k in range(1, POOL):
            u = synth.stereo_unit(w, h, 300 + d, rvec=r * k, tvec=t * k)
            fr.append((u["l1"], u["r1"]))
        out.append((base["P_l"], base["P_r"], fr))
    return out


def frame(drv, k):
    """frame k of a drive that replays its pool back and forth"""
    period = 2 * (POOL - 1)
    j = k % period
    return drv[2][j if j < POOL else period - j]


def run(ctx, plan, n_slots, opened):
    """plan: per submission k (from 1), {slot: (drive, frame index)}; opened: starts at frame index 0 (vo_mseq_open),
    else consecutive begins (a frame index 0 in every slot of a submission begins a batch).  Returns the per-mode
    numbers."""
    steps = len(plan)
    t_step, starts_at, launches = [], [], {True: [], False: []}
    done = 0

    cur = [n_slots]                                 # sequences of the running batch (the last one may hold fewer)

    def pairs(k):
        if not opened and any(j == 0 for _, j in plan[k].values()):
            cur[0] = len(plan[k])
        lefts, rights, start = [None] * cur[0], [None] * cur[0], {}
        for q, (drv, j) in plan[k].items():
            lefts[q], rights[q] = frame(drv, j)
            if j == 0:
                start[q] = (drv[0], drv[1])
        return lefts, rights, start

    def submit(k):
        lefts, rights, start = pairs(k)
        l0 = ctx.kernel_launches()
        if not opened and start:
            ctx.mseq_begin(lefts, rights, np.stack([v[0] for v in start.values()]), np.stack([v[1] for v in start.values()]))
            return False
        ctx.mseq_submit(lefts, rights, start=start or None)
        launches[bool(start)].append(ctx.kernel_launches() - l0)
        return True

    t0 = time.perf_counter()
    k = 0
    inflight = []
    last = t0
    live = 0
    while k < steps or inflight:
        while k < steps and len(inflight) < 2:
            if not opened and any(j == 0 for _, j in plan[k].values()):
                if inflight:                        # a begin ends the run: wait for what is in flight first
                    break
                submit(k)
            else:
                submit(k)
                inflight.append(k)
            k += 1
        if not inflight:
            continue
        kk = inflight.pop(0)
        ctx.mseq_wait(want_points=False)
        now = time.perf_counter()
        t_step.append(now - last)
        starts_at.append(opened and any(j == 0 for _, j in plan[kk].values()))
        last = now
        done += sum(1 for _, j in plan[kk].values() if j > 0)
        live += len(plan[kk])
    wall = time.perf_counter() - t0
    subs = len(t_step)
    live /= max(subs, 1)
    st = [t for t, s in zip(t_step, starts_at) if s]
    pl = [t for t, s in zip(t_step, starts_at) if not s]
    return dict(fps=done / wall, submissions=subs, mean_live=live,
                step_ms_start=1e3 * statistics.median(st) if st else None,
                step_ms_plain=1e3 * statistics.median(pl) if pl else None,
                launches_plain=statistics.median(launches[False]) if launches[False] else None,
                launches_start=max(launches[True]) if launches[True] else None)


def plans(drv, lengths, n):
    """(opened plan, batches plan) of the queue through n slots"""
    sched = queue_schedule(lengths, n)
    steps = max(k0 + L - 1 for (_, k0), L in zip(sched, lengths))
    opened = [dict() for _ in range(steps)]
    for d, ((q, k0), L) in enumerate(zip(sched, lengths)):
        for j in range(L):
            opened[k0 - 1 + j][q] = (drv[d], j)
    batches = []
    for i in range(0, len(lengths), n):
        group = list(range(i, min(i + n, len(lengths))))
        for j in range(max(lengths[g] for g in group)):
            batches.append({q: (drv[g], j) for q, g in enumerate(group) if j < lengths[g]})
    return opened, batches


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=float, default=0.01)
    ap.add_argument("--size", default="640x240")
    ap.add_argument("--slots", default="2,4,8")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json")
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    counts = [int(v) for v in a.slots.split(",")]
    if a.check:
        for n in counts:
            sched = queue_schedule(KITTI_LENGTHS, n)
            qs = max(k0 + L - 1 for (_, k0), L in zip(sched, KITTI_LENGTHS))
            bs = sum(max(KITTI_LENGTHS[i:i + n]) for i in range(0, len(KITTI_LENGTHS), n))
            print(f"N = {n}: starts {qs} submissions ({sum(KITTI_LENGTHS) / qs:.1f} live), "
                  f"batches {bs - len(range(0, len(KITTI_LENGTHS), n))} submissions "
                  f"({(sum(KITTI_LENGTHS) - len(KITTI_LENGTHS)) / (bs - len(range(0, len(KITTI_LENGTHS), n))):.1f} live)")
        return
    from mseq_timing import card
    from visual_odom_b200.capi import Context
    w, h = (int(v) for v in a.size.split("x"))
    lengths = [max(3, round(L * a.scale)) for L in KITTI_LENGTHS]
    drv = drives(w, h, len(lengths))
    ctx = Context(0, max_features=4096)
    out = dict(card=card(), size=[w, h], lengths=lengths, modes={})
    for n in counts:
        opened, batches = plans(drv, lengths, n)
        res = {"start": [], "batches": []}
        for r in range(a.rounds + 1):                   # round 0 warms up (graph captures)
            ctx.mseq_open(n, w, h)
            s = run(ctx, opened, n, True)
            b = run(ctx, batches, n, False)
            if r:
                res["start"].append(s); res["batches"].append(b)
        for mode, rs in res.items():
            m = {k: statistics.median(x[k] for x in rs) if rs[0][k] is not None else None for k in rs[0]}
            out["modes"][f"N={n} {mode}"] = m
    # idle slots: 8 opened slots with 2 live drives, against vo_mseq_begin of the 2
    L = max(lengths)
    live2 = [{q: (drv[q], j) for q in range(2)} for j in range(L)]
    res = {"open 8, 2 live": [], "begin 2": []}
    for r in range(a.rounds + 1):
        ctx.mseq_open(8, w, h)
        s = run(ctx, live2, 8, True)
        b = run(ctx, live2, 2, False)
        if r:
            res["open 8, 2 live"].append(s); res["begin 2"].append(b)
    for mode, rs in res.items():
        out["modes"][f"idle {mode}"] = {k: statistics.median(x[k] for x in rs) if rs[0][k] is not None else None for k in rs[0]}
    ctx.close()
    print(f"card (name, power limit, max SM clock): {out['card']}")
    print(f"{w}x{h}, queue lengths {lengths}")
    print(f"{'mode':<22} {'frames/s':>9} {'subs':>6} {'live':>5} {'step start ms':>14} {'step plain ms':>14} {'launch plain':>13} {'launch start':>13}")
    f = lambda v, fmt: "-" if v is None else format(v, fmt)
    for name, m in out["modes"].items():
        print(f"{name:<22} {m['fps']:>9.0f} {m['submissions']:>6.0f} {m['mean_live']:>5.2f} {f(m['step_ms_start'], '.3f'):>14} "
              f"{f(m['step_ms_plain'], '.3f'):>14} {f(m['launches_plain'], '.0f'):>13} {f(m['launches_start'], '.0f'):>13}")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
