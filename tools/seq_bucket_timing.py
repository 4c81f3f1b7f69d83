#!/usr/bin/env python
"""Cost and accuracy of denser bucketing (vo_params.features_per_bucket) in the streaming sequence modes, on the GPU.

    python tools/seq_bucket_timing.py [--frames 40] [--rounds 5] [--n-seq 8] [--k 1,2,4,8] [--json out.json]

On the synthetic 1241x376 drive (synth.stereo_unit, the motion of tests/test_gpu_seq.py) one context per
features_per_bucket value k (bucket_rows_divisor 10) runs the same frames, the k values alternated round by round, and
reports per k and per mode (vo_seq_* with one sequence, vo_mseq_* with --n-seq sequences):
  - pipelined frames/s: submit / wait with two frames in flight (vo_mseq_*: stereo frames of all sequences per second)
  - one-push latency: median wall time of one synchronous submission (submit + wait)
  - features fed per frame: the record's n_features (the bucketed points that enter the LK ring), mean over the frames
  - kernel launches per submission (vo_kernel_launches)
  - the final translation error of the single-sequence run's frame_pose against the drive's rendered motion (each frame
    is drawn at X_k = R(k r) X_0 + k t, so the step from frame k - 1 is [R(r) | k t - (k - 1) R(r) t]), integrated with
    the reference's rule, in metres and as a share of the path length
Median of the rounds, with min and max.  The card's name, power limit and max SM clock are printed with the numbers;
they are part of them."""
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
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
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


def true_pose(n):
    """frame_pose after n frames of the rendered motion, integrated as the reference integrates the PnP's [R|t]."""
    import cv2
    from oracle import ref_path
    R, _ = cv2.Rodrigues(STEP_R.reshape(3, 1))
    pose = np.eye(4)
    for k in range(1, n + 1):
        pose = ref_path.integrate_pose(pose, R, k * STEP_T - (k - 1) * (R @ STEP_T))
    return pose


def run(ctx, base, fr, n_seq, pipelined):
    """One pass over the drive: (frames/s or per-submission latencies, mean n_features, launches per submission)."""
    multi = n_seq > 1
    if multi:
        ctx.mseq_begin([fr[0][0]] * n_seq, [fr[0][1]] * n_seq, base["P_l"], base["P_r"])
        submit = lambda k: ctx.mseq_submit([fr[k][0]] * n_seq, [fr[k][1]] * n_seq)
        wait = lambda: ctx.mseq_wait(want_points=False)[0]
    else:
        ctx.seq_begin(fr[0][0], fr[0][1], base["P_l"], base["P_r"])
        submit = lambda k: ctx.seq_submit(*fr[k])
        wait = lambda: ctx.seq_wait(want_points=False)
    l0 = ctx.kernel_launches()
    feats, lat = [], []
    t0 = time.perf_counter()
    if pipelined:
        submit(1)
        for k in range(1, len(fr)):
            if k + 1 < len(fr):
                submit(k + 1)
            feats.append(wait()["n_features"])
    else:
        for k in range(1, len(fr)):
            t1 = time.perf_counter()
            submit(k)
            feats.append(wait()["n_features"])
            lat.append(time.perf_counter() - t1)
    dt = time.perf_counter() - t0
    rate = n_seq * (len(fr) - 1) / dt if pipelined else float(np.median(lat))
    return rate, float(np.mean(feats)), (ctx.kernel_launches() - l0) / (len(fr) - 1)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--n-seq", type=int, default=8)
    ap.add_argument("--k", default="1,2,4,8", help="features_per_bucket values")
    ap.add_argument("--json", help="also write the result here")
    a = ap.parse_args()
    from visual_odom_b200 import capi
    ks = [int(x) for x in a.k.split(",")]
    base, fr = frames(1241, 376, a.frames + 1)
    modes = (("seq", 1), ("mseq", a.n_seq))
    ctxs = {k: capi.Context(0, max_features=4096, features_per_bucket=k) for k in ks}
    res = {(k, m): dict(fps=[], lat=[], feats=[], launches=[]) for k in ks for m, _ in modes}
    err = {}
    for k in ks:                                      # warm-up: captures every graph once; the accuracy pass
        for _, n in modes:
            run(ctxs[k], base, fr[:4], n, True)
        run(ctxs[k], base, fr, 1, True)
        err[k] = float(np.linalg.norm(ctxs[k].seq_pose()[:3, 3] - true_pose(a.frames)[:3, 3]))
    for _ in range(a.rounds):
        for k in ks:
            for m, n in modes:
                fps, feats, launches = run(ctxs[k], base, fr, n, True)
                lat, _, _ = run(ctxs[k], base, fr, n, False)
                r = res[(k, m)]
                r["fps"].append(fps); r["lat"].append(lat); r["feats"].append(feats); r["launches"].append(launches)
    for c in ctxs.values():
        c.close()
    path = a.frames * float(np.linalg.norm(STEP_T))
    out = dict(card=card(), image="1241x376", bucket_rows_divisor=10, frames=a.frames, rounds=a.rounds, n_seq=a.n_seq,
               rows=[])
    for k in ks:
        for m, n in modes:
            r = res[(k, m)]
            out["rows"].append(dict(k=k, mode=m, n_seq=n, fps=float(np.median(r["fps"])), fps_min=float(np.min(r["fps"])),
                                    fps_max=float(np.max(r["fps"])), latency_ms=1e3 * float(np.median(r["lat"])),
                                    latency_ms_min=1e3 * float(np.min(r["lat"])), latency_ms_max=1e3 * float(np.max(r["lat"])),
                                    features_per_frame=float(np.median(r["feats"])),
                                    launches_per_submission=float(np.median(r["launches"])),
                                    final_translation_error_m=err[k], final_translation_error_share=err[k] / path))
    print(f"card (name, power limit, max SM clock): {out['card']}")
    print("| k | mode | frames/s [min, max] | one-push latency ms [min, max] | features / frame | launches / submission "
          "| final translation error |")
    print("|---|---|---|---|---|---|---|")
    for o in out["rows"]:
        print(f"| {o['k']} | {o['mode']} x{o['n_seq']} | {o['fps']:.0f} [{o['fps_min']:.0f}, {o['fps_max']:.0f}] "
              f"| {o['latency_ms']:.3f} [{o['latency_ms_min']:.3f}, {o['latency_ms_max']:.3f}] | {o['features_per_frame']:.0f} "
              f"| {o['launches_per_submission']:.0f} | {o['final_translation_error_m']:.3f} m "
              f"({100 * o['final_translation_error_share']:.2f} %) |")
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
