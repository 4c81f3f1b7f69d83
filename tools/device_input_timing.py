#!/usr/bin/env python
"""Images from host memory against images already on the GPU, measured on the GPU.

    python tools/device_input_timing.py [--frames 60] [--rounds 5] [--steps 60] [--parent DIR] [--json out.json]

On the synthetic 1241x376 drive (synth.stereo_unit, the motion of tests/test_gpu_seq.py), alternated round by round, median
over rounds:
  - sequence mode, per input kind (pinned-host gray, device gray, pinned-host BGR, device BGR HWC, device RGB CHW):
    pipelined frames/s (two frames in flight) and the one-push latency (median wall time of submit + wait);
  - the batched e2e loop: 8 units x 2000 features per submission, three submissions in flight, with pinned-host images
    (vo_batch_submit) against device images (vo_batch_submit_device); units/s.
Device inputs are submitted on a torch stream the context is pointed at.  With --parent DIR (a built checkout of another
commit) the pinned-host BGR sequence row is also timed with that checkout's library, in child processes alternated with
this one's.  The card's name, power limit and max SM clock are printed with the numbers; they are part of them."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

STEP_R = np.array([0.001, -0.004, 0.0005])
STEP_T = np.array([0.01, -0.003, -0.2])
SEQ_ROWS = ("host_gray", "dev_gray", "host_bgr", "dev_bgr_hwc", "dev_rgb_chw")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown (nvidia-smi unavailable)"


def colourise(gray, seed):
    rng = np.random.default_rng(seed)
    tint = rng.integers(-20, 21, gray.shape + (3,))
    return np.clip(gray[..., None].astype(np.int32) + tint, 0, 255).astype(np.uint8)


def seq_inputs(row, n, torch):
    """(P_l, P_r, frames): the frames of `row` as pinned numpy arrays or CUDA tensors."""
    from visual_odom_b200 import synth
    base = synth.stereo_unit(1241, 376, 31)
    gray = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(1241, 376, 31, rvec=STEP_R * k, tvec=STEP_T * k)
        gray.append((u["l1"], u["r1"]))
    imgs = gray if row.endswith("gray") else [(colourise(l, 2 * i), colourise(r, 2 * i + 1)) for i, (l, r) in enumerate(gray)]
    if row == "dev_rgb_chw":
        imgs = [tuple(np.ascontiguousarray(a[..., ::-1].transpose(2, 0, 1)) for a in p) for p in imgs]
    if row.startswith("host"):
        out = [tuple(torch.from_numpy(a).pin_memory().numpy() for a in p) for p in imgs]
    else:
        out = [tuple(torch.from_numpy(a).cuda() for a in p) for p in imgs]
    return base["P_l"], base["P_r"], out


def seq_calls(ctx, row):
    """(begin, submit, push) of `row`."""
    if row.startswith("host"):
        if row == "host_bgr":
            return ctx.seq_begin_bgr, ctx.seq_submit, lambda l, r: ctx.seq_push_ptr(l.ctypes.data, r.ctypes.data, l.strides[0], 3)
        return ctx.seq_begin, ctx.seq_submit, lambda l, r: ctx.seq_push(l, r, want_points=False)
    order = None if row == "dev_gray" else "rgb" if "rgb" in row else "bgr"
    return (lambda l, r, P_l, P_r: ctx.seq_begin_device(l, r, P_l, P_r, order=order),
            lambda l, r: ctx.seq_submit_device(l, r, order=order),
            lambda l, r: ctx.seq_push_device(l, r, order=order, want_points=False))


def time_seq(ctx, row, data):
    P_l, P_r, fr = data
    begin, submit, push = seq_calls(ctx, row)
    begin(fr[0][0], fr[0][1], P_l, P_r)
    t0 = time.perf_counter()
    submit(*fr[1])
    for k in range(1, len(fr)):
        if k + 1 < len(fr):
            submit(*fr[k + 1])
        ctx.seq_wait(want_points=False)
    fps = (len(fr) - 1) / (time.perf_counter() - t0)
    begin(fr[0][0], fr[0][1], P_l, P_r)
    lat = []
    for l, r in fr[1:]:
        t0 = time.perf_counter()
        push(l, r)
        lat.append(time.perf_counter() - t0)
    return fps, float(np.median(lat))


def batch_inputs(device, torch, n_units=8):
    from visual_odom_b200 import synth
    units = []
    for i in range(n_units):
        u = synth.stereo_unit(1241, 376, 100 + i)
        imgs = {k: (torch.from_numpy(u[k]).cuda() if device else torch.from_numpy(u[k]).pin_memory().numpy()) for k in ("l0", "r0", "l1", "r1")}
        units.append(dict(imgs, n_select=2000, t_prev=(0.0, 0.0, -0.8)))
    return units, u["P_l"], u["P_r"]


def time_batch(ctx, device, units, steps, depth=3):
    """units/s over `steps` waited submissions of the same units with `depth` submissions in flight."""
    B = len(units)
    if device:
        def submit(s):
            ctx.batch_submit_device(units, (s % depth) * B)
    else:
        arr, keep, pitch = ctx.make_units(units)

        def submit(s):
            ctx.batch_submit(arr, (s % depth) * B, pitch)
    for s in range(depth):
        submit(s)
    t0 = time.perf_counter()
    for s in range(steps):
        ctx.batch_wait((s % depth) * B, B, raw=True)
        submit(s + depth)
    dt = time.perf_counter() - t0
    for s in range(steps, steps + depth):
        ctx.batch_wait((s % depth) * B, B, raw=True)
    return steps * B / dt


def child(a):
    """One round of the pinned-host BGR row with the library under --root (for --parent comparisons)."""
    sys.path.insert(0, os.path.abspath(a.root))
    import torch
    from visual_odom_b200 import capi
    ctx = capi.Context(0, max_features=4096, max_units=2)
    data = seq_inputs("host_bgr", a.frames + 1, torch)
    time_seq(ctx, "host_bgr", (data[0], data[1], data[2][:4]))     # graphs captured, untimed
    fps, lat = time_seq(ctx, "host_bgr", data)
    print(json.dumps(dict(fps=fps, lat=lat)))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=60, help="waited submissions per batched round")
    ap.add_argument("--parent", help="built checkout whose host-BGR sequence row is timed alongside")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--json", help="also write the result here")
    a = ap.parse_args()
    if a.child:
        return child(a)
    sys.path.insert(0, os.path.abspath(a.root))
    import torch
    from visual_odom_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    out = dict(card=card(), image="1241x376", frames=a.frames, rounds=a.rounds)
    print(f"card (name, power limit, max SM clock): {out['card']}", flush=True)

    ctx = capi.Context(0, max_features=4096, max_units=2)
    s = torch.cuda.Stream()
    res = {r: dict(fps=[], lat=[]) for r in SEQ_ROWS}
    with torch.cuda.stream(s):
        data = {r: seq_inputs(r, a.frames + 1, torch) for r in SEQ_ROWS}
        for r in SEQ_ROWS:                                       # graphs captured, untimed
            time_seq(ctx, r, (data[r][0], data[r][1], data[r][2][:4]))
        for _ in range(a.rounds):
            for r in SEQ_ROWS:
                fps, lat = time_seq(ctx, r, data[r])
                res[r]["fps"].append(fps); res[r]["lat"].append(lat)
    ctx.close()
    for r in SEQ_ROWS:
        out[r] = dict(pipelined_fps=float(np.median(res[r]["fps"])), push_latency_ms=1e3 * float(np.median(res[r]["lat"])))
        print(f"sequence {r:12s}: pipelined {out[r]['pipelined_fps']:.0f} frames/s, one-push latency "
              f"{out[r]['push_latency_ms']:.3f} ms", flush=True)

    ctx = capi.Context(0, max_features=2048, max_units=24)
    bres = {"host_pinned": [], "device": []}
    with torch.cuda.stream(s):
        hu, P_l, P_r = batch_inputs(False, torch)
        du, _, _ = batch_inputs(True, torch)
        ctx.batch_configure(1241, 376, 3 * len(hu), P_l, P_r)
        ctx.set_option("batch_outputs", 1)
        for dev, units in ((False, hu), (True, du)):
            time_batch(ctx, dev, units, 6)                          # warm-up
        for _ in range(a.rounds):
            for name, dev, units in (("host_pinned", False, hu), ("device", True, du)):
                bres[name].append(time_batch(ctx, dev, units, a.steps))
    ctx.close()
    for name in bres:
        out["batch_e2e_" + name] = dict(units_per_s=float(np.median(bres[name])))
        print(f"batched e2e (8 units x 2000 features, 3 in flight) {name:11s}: {out['batch_e2e_' + name]['units_per_s']:.0f} units/s",
              flush=True)

    if a.parent:
        rows = {"this": [], "parent": []}
        for _ in range(a.rounds):
            for name, root in (("this", a.root), ("parent", a.parent)):
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--root", root, "--frames", str(a.frames)],
                                   capture_output=True, text=True, check=True)
                rows[name].append(json.loads(r.stdout.strip().splitlines()[-1]))
        for name in rows:
            out["host_bgr_" + name] = dict(pipelined_fps=float(np.median([x["fps"] for x in rows[name]])),
                                           push_latency_ms=1e3 * float(np.median([x["lat"] for x in rows[name]])))
            print(f"sequence host_bgr ({name:6s} commit, own process): pipelined {out['host_bgr_' + name]['pipelined_fps']:.0f} "
                  f"frames/s, one-push latency {out['host_bgr_' + name]['push_latency_ms']:.3f} ms", flush=True)
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
