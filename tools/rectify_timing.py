#!/usr/bin/env python
"""Rectification on against off in the multi-sequence mode (vo_mseq_rectify), alternated round by round:

    python tools/rectify_timing.py [--steps 60] [--rounds 3] [--out DIR]

For n_seq = 1, 8 and 32 sequences of one synthetic drive, from host gray and from device gray input, at 1241 x 376 and
752 x 480: frames/s and step time of pipelined submissions (two in flight) with every slot rectified on raw frames ("on"),
and with every slot plain on the same frames rectified beforehand ("off": the same images reach the tracker, so the
difference is what rectification costs).  Then the remap alone: the launch is internal to a submission, so it cannot
be bracketed with CUDA events from outside; one torch.profiler run (CUDA activities, in a run of its own) of rectified
host submissions gives the device time of each k_bgr_to_gray launch, whose bytes (maps 6 B/px, a staged gray image
1 B/px read, 1 B/px written, per image) are set against the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same run and printed with the
numbers; the JSON goes to DIR/rectify_timing.json."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

# the rig of each size: EuRoC's at its own 752 x 480, the KITTI-raw-like pair at 1241 x 376
RIGS = {(1241, 376): ("kitti_raw_left", "kitti_raw_right"), (752, 480): ("euroc_cam0", "euroc_cam1")}

def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable ({e})"
    return q


def frames(w, h, n=8):
    from visual_odom_b200 import synth
    base = synth.stereo_unit(w, h, 3)
    fr = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, 3, rvec=np.array((0.001, -0.003, 0.0005)) * k, tvec=np.array((0.01, -0.002, -0.2)) * k)
        fr.append((u["l1"], u["r1"]))
    return base["P_l"], base["P_r"], fr


def rig(w, h):
    from visual_odom_b200 import synth
    return synth.rectify_rig(*RIGS[(w, h)])


def prerectified(ctx, fr, rect, w, h):
    """The frames as the library rectifies them (vo_remap, which is cv2.remap bit for bit)."""
    from visual_odom_b200 import capi
    maps = [capi.rectify_maps(tuple(rect[s]), w, h) for s in ("left", "right")]
    return [tuple(ctx.remap(img, *maps[k]) for k, img in enumerate(p)) for p in fr]


def run(ctx, n, P_l, P_r, fr, rect, device, steps):
    """Seconds per pipelined step of n sequences (after 2 warm-up steps)."""
    import torch
    ctx.mseq_rectify(0, [rect] * n)
    ctx.mseq_begin([fr[0][0]] * n, [fr[0][1]] * n, P_l, P_r)
    if device:
        dfr = [[torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in p] for p in fr]

    def submit(k):
        p = (dfr if device else fr)[1 + k % (len(fr) - 1)]
        if device:
            ctx.mseq_submit_device([p[0]] * n, [p[1]] * n)
        else:
            ctx.mseq_submit([p[0]] * n, [p[1]] * n)
    submit(0)
    for k in range(1, 3):
        submit(k); ctx.mseq_wait(want_points=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(3, 3 + steps):
        submit(k); ctx.mseq_wait(want_points=False)
    ctx.mseq_wait(want_points=False)
    dt = (time.perf_counter() - t0) / steps
    ctx.mseq_rectify(0, [None] * n)
    return dt


def remap_kernel_times(ctx, w, h, n, P_l, P_r, fr, rect):
    import torch
    from torch.profiler import profile, ProfilerActivity
    ctx.mseq_rectify(0, [rect] * n)
    ctx.mseq_begin([fr[0][0]] * n, [fr[0][1]] * n, P_l, P_r)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(1, len(fr)):
            ctx.mseq_submit([fr[k][0]] * n, [fr[k][1]] * n); ctx.mseq_wait(want_points=False)
        torch.cuda.synchronize()
    ctx.mseq_rectify(0, [None] * n)
    us = [e.device_time for e in prof.events() if "k_bgr_to_gray" in e.name and e.device_time > 0]
    px = 2 * n * w * h
    b = px * (6 + 1 + 1)
    t = float(np.median(us)) * 1e-6 if us else float("nan")
    return dict(n_seq=n, launches=len(us), us_per_launch=t * 1e6, bytes=b, tb_s=b / t / 1e12,
                share_of_3_35_tb_s=b / t / 3.35e12)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="1241x376,752x480")
    ap.add_argument("--nseq", default="1,8,32")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from visual_odom_b200.capi import Context
    out = dict(card=card(), rows=[], remap=[])
    print("card (name, power limit, max SM clock):", out["card"])
    ctx = Context(0, max_features=8192, max_units=2)
    for size in a.sizes.split(","):
        w, h = (int(v) for v in size.split("x"))
        P_l, P_r, fr = frames(w, h)
        rect = rig(w, h)
        fr_rect = prerectified(ctx, fr, rect, w, h)
        for n in (int(v) for v in a.nseq.split(",")):
            for device in (False, True):
                t = {False: [], True: []}
                for r in range(a.rounds):
                    for on in ((False, True) if r % 2 == 0 else (True, False)):
                        t[on].append(run(ctx, n, P_l, P_r, fr if on else fr_rect, rect if on else None, device, a.steps))
                off, on = float(np.median(t[False])), float(np.median(t[True]))
                row = dict(w=w, h=h, n_seq=n, input="device" if device else "host", step_ms_off=off * 1e3,
                           step_ms_on=on * 1e3, fps_off=n / off, fps_on=n / on, rounds=a.rounds, steps=a.steps)
                out["rows"].append(row)
                print(f"{w}x{h} n_seq={n:2d} {row['input']:6s}: off {off * 1e3:7.3f} ms/step {n / off:8.0f} frames/s | "
                      f"on {on * 1e3:7.3f} ms/step {n / on:8.0f} frames/s")
        for n in (1, 8, 32):
            k = remap_kernel_times(ctx, w, h, n, P_l, P_r, fr, rect)
            k.update(w=w, h=h)
            out["remap"].append(k)
            print(f"{w}x{h} remap launch, {2 * n} images: {k['us_per_launch']:.1f} us, {k['tb_s']:.2f} TB/s "
                  f"({100 * k['share_of_3_35_tb_s']:.0f} % of 3.35 TB/s)")
    # host time of a rectified begin: the same begin with and without rectification (maps of both cameras + their copy)
    w, h = 1241, 376
    P_l, P_r, fr = frames(w, h, 2)
    rect = rig(w, h)
    tb = {False: [], True: []}
    for r in range(6):
        on = r % 2 == 1
        ctx.mseq_rectify(0, [rect if on else None])
        t0 = time.perf_counter()
        ctx.mseq_begin([fr[0][0]], [fr[0][1]], P_l, P_r)
        tb[on].append(time.perf_counter() - t0)
    ctx.mseq_rectify(0, [None])
    out["begin_ms_1241x376"] = {"plain": float(np.median(tb[False])) * 1e3, "rectified": float(np.median(tb[True])) * 1e3}
    print(f"a one-sequence begin at 1241x376: {out['begin_ms_1241x376']['plain']:.1f} ms plain, "
          f"{out['begin_ms_1241x376']['rectified']:.1f} ms rectified (host wall time)")
    ctx.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "rectify_timing.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
