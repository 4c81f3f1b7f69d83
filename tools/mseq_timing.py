#!/usr/bin/env python
"""Scaling of the multi-sequence streaming mode (vo_mseq_*) with the number of sequences, measured on the GPU.

    python tools/mseq_timing.py [--frames 40] [--rounds 5] [--counts 1,2,4,8,16,32] [--mono-rotation] [--mixed-calibration]
                                [--mixed-sizes] [--device-input] [--device-results] [--mixed-params] [--json out.json]

Synthetic 1241x376 drives (synth.stereo_unit; eight seeds, each with its own motion) of `--frames` frames each;
sequence q replays drive q % 8, forwards for even q // 8 and backwards for odd, so up to 16 sequences are distinct and
larger counts repeat them (the work per sequence is the same either way).  One context runs, alternated round by round:
  - "seq": the single-sequence mode, vo_seq_submit / vo_seq_wait with two frames in flight
  - n_seq = each count: vo_mseq_submit / vo_mseq_wait with two submissions in flight
and reports per mode the median over the rounds of the aggregate frames/s (sequence-frames per second of wall time), the
per-step latency (wall time per submission in the pipelined loop) and the kernel launches per submission
(vo_kernel_launches).  `--mono-rotation` runs every mode twice per round, without and with trackingFrame2Frame's
mono_rotation branch (the option "mono_rotation" for vo_seq_*, the flag VO_MSEQ_MONO_ROTATION for vo_mseq_*), and
reports both.  `--mixed-calibration` also runs every vo_mseq_* count with one calibration per sequence
(vo_mseq_begin_calib): sequence q is then rendered with, and run with, its own camera (focal length, principal point and
baseline spread over +-10 %, +-20 px and +-15 %), so that no two sequences share a calibration; the motions are those
of the one-calibration run.  Both are timed in the same rounds, alternated.  `--mixed-sizes` (counts 3, 11 and 32 unless
--counts is given) also runs every vo_mseq_* count with sequence q at the image size of KITTI odometry training sequence
q mod 11 (1241x376 for 00-02, 1242x375 for 03, 1226x370 for 04-10: the 3 : 1 : 7 mix of the training set, through
vo_mseq_begin_sized), the drives rendered at those sizes with the motions of the one-size run, timed against the same
count all at 1241x376 in the same rounds, alternated.  `--device-input` (counts 1, 8, 16 and 32 unless --counts is given)
times every vo_mseq_* count three ways in the same rounds, alternated: host gray images (vo_mseq_submit, the loop above),
and every frame made resident as CUDA tensors before the timed window and fed through vo_mseq_submit_device as gray
(H, W) and as BGR (H, W, 3) tensors; it also times the host side of one vo_mseq_submit_device call (the binding, and the
C call alone) at 32 and 64 sequences.  `--device-results` (counts 1, 8 and 32 unless --counts is given) times every
vo_mseq_* count two ways in the same rounds, alternated, both with resident gray CUDA tensors through
vo_mseq_submit_device: host waits that return the point lists (vo_mseq_wait with pts4), and a run begun with
VO_MSEQ_DEVICE_RESULTS whose waits are vo_mseq_wait_device into one reused set of CUDA tensors, each followed by a trivial
torch consumer of them on the same stream (the loop ends with a synchronise, inside the timed window).  It adds the host
time per step spent inside the submit and wait calls, and the kernel launches per submission and per wait.
`--mixed-params` (counts 1, 8 and 32 unless --counts is given) also runs every vo_mseq_* count with one set of tracking
parameters per sequence (vo_mseq_params: sequence q takes set q mod 8 of PARAM_SETS, FAST thresholds, LK criteria, PnP
settings, bucket grids and densities), timed against the same count at the context's one set in the same rounds,
alternated.  The card's name, power limit and max SM clock, read in the same run, are printed with the numbers;
they are part of them."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

W, H, DRIVES = 1241, 376, 8
KITTI_SIZES = [(1241, 376)] * 3 + [(1242, 375)] + [(1226, 370)] * 7      # training sequences 00 .. 10


# --mixed-params: sequence q runs with PARAM_SETS[q % 8] (every bound within max_features = 4096 at 1241x376)
PARAM_SETS = [dict(), dict(fast_threshold=12), dict(features_per_bucket=3, bucket_rows_divisor=6),
              dict(lk_max_iters=7, lk_epsilon=0.05, lk_min_eig=1e-2), dict(pnp_iterations=40, pnp_reproj_error=1.5, pnp_confidence=0.99),
              dict(refill_threshold=500, bucket_age_threshold=3, circ_threshold=1), dict(fast_threshold=30, lk_max_iters=15),
              dict(features_per_bucket=2, bucket_rows_divisor=12)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown (nvidia-smi unavailable)"


def motion(d):
    rng = np.random.default_rng(100 + d)
    return rng.uniform(-0.004, 0.004, 3) * np.array([1.0, 1.0, 0.25]), np.array([0.0, 0.0, -0.2]) + rng.uniform(-0.02, 0.02, 3)


def calibration(q, n):
    """the camera of sequence q of n in the mixed-calibration runs (KITTI 00's, spread over the sequences)"""
    from visual_odom_b200 import synth
    f = -1.0 + 2.0 * q / max(n - 1, 1)                # -1 .. 1
    c = synth.KITTI00
    return dict(fx=c["fx"] * (1 + 0.1 * f), fy=c["fy"] * (1 + 0.1 * f), cx=c["cx"] + 20 * f, cy=c["cy"] - 20 * f,
                bf=c["bf"] * (1 - 0.15 * f))


def render(job):
    from visual_odom_b200 import synth
    d, k, cal, (w, h) = job
    r, t = motion(d)
    u = synth.stereo_unit(w, h, 50 + d, rvec=r * k, tvec=t * k, **({} if cal is None else dict(cal=cal)))
    return (u["l0"], u["r0"]) if k == 0 else (u["l1"], u["r1"])


def drives(n_frames, cals=None, size=(W, H)):
    """[drive][frame] = (left, right) of size w x h, rendered in parallel (one synth call per frame).  cals: one
    calibration per drive (drive i then replays the motion of drive i % DRIVES), else DRIVES drives at KITTI 00's."""
    ids = [(d, None) for d in range(DRIVES)] if cals is None else [(i % DRIVES, c) for i, c in enumerate(cals)]
    jobs = [(d, k, c, size) for d, c in ids for k in range(n_frames)]
    with ProcessPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        pairs = list(ex.map(render, jobs, chunksize=4))
    return [pairs[i * n_frames:(i + 1) * n_frames] for i in range(len(ids))]


def sequence(dr, q):
    fr = dr[q % DRIVES]
    return fr if (q // DRIVES) % 2 == 0 else fr[::-1]


def run_seq(ctx, P_l, P_r, fr, mono=False):
    ctx.set_option("mono_rotation", 1 if mono else 0)
    ctx.seq_begin(fr[0][0], fr[0][1], P_l, P_r)
    ctx.set_option("mono_rotation", 0)             # the sequence keeps the value it was begun with
    l0 = ctx.kernel_launches()
    t0 = time.perf_counter()
    ctx.seq_submit(*fr[1])
    for k in range(1, len(fr)):
        if k + 1 < len(fr):
            ctx.seq_submit(*fr[k + 1])
        ctx.seq_wait(want_points=False, mono=mono)
    dt = time.perf_counter() - t0
    steps = len(fr) - 1
    return steps / dt, dt / steps, (ctx.kernel_launches() - l0) / steps


def run_mseq(ctx, P_l, P_r, seqs, mono=False):
    n, nf = len(seqs), len(seqs[0])
    ctx.mseq_begin([s[0][0] for s in seqs], [s[0][1] for s in seqs], P_l, P_r, mono_rotation=mono)
    frame = [([s[k][0] for s in seqs], [s[k][1] for s in seqs]) for k in range(nf)]
    l0 = ctx.kernel_launches()
    t0 = time.perf_counter()
    ctx.mseq_submit(*frame[1])
    for k in range(1, nf):
        if k + 1 < nf:
            ctx.mseq_submit(*frame[k + 1])
        ctx.mseq_wait(want_points=False, mono=mono)
    dt = time.perf_counter() - t0
    steps = nf - 1
    return n * steps / dt, dt / steps, (ctx.kernel_launches() - l0) / steps


def run_mseq_device(ctx, P_l, P_r, seqs, order=None):
    """run_mseq with every frame a CUDA tensor (resident before the timed window) through vo_mseq_submit_device"""
    n, nf = len(seqs), len(seqs[0])
    ctx.mseq_begin_device([s[0][0] for s in seqs], [s[0][1] for s in seqs], P_l, P_r, order=order)
    frame = [([s[k][0] for s in seqs], [s[k][1] for s in seqs]) for k in range(nf)]
    l0 = ctx.kernel_launches()
    t0 = time.perf_counter()
    ctx.mseq_submit_device(*frame[1], order=order)
    for k in range(1, nf):
        if k + 1 < nf:
            ctx.mseq_submit_device(*frame[k + 1], order=order)
        ctx.mseq_wait(want_points=False)
    dt = time.perf_counter() - t0
    steps = nf - 1
    return n * steps / dt, dt / steps, (ctx.kernel_launches() - l0) / steps


def run_mseq_dres(ctx, P_l, P_r, seqs, device_results):
    """device input, two submissions in flight; host waits with point lists, or vo_mseq_wait_device + a torch consumer.
    Returns (aggregate frames/s, step time, host time per step in the calls, launches per submission, per wait)."""
    import torch
    n, nf = len(seqs), len(seqs[0])
    ctx.mseq_begin_device([s[0][0] for s in seqs], [s[0][1] for s in seqs], P_l, P_r, device_results=device_results)
    frame = [([s[k][0] for s in seqs], [s[k][1] for s in seqs]) for k in range(nf)]
    out = ctx.mseq_dresults_alloc() if device_results else None
    acc = torch.zeros((), dtype=torch.float64, device="cuda")
    host, l_sub, l_wait = 0.0, 0, 0

    def submit(k):
        nonlocal host, l_sub
        l, t = ctx.kernel_launches(), time.perf_counter()
        ctx.mseq_submit_device(*frame[k])
        host += time.perf_counter() - t
        l_sub += ctx.kernel_launches() - l
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    submit(1)
    for k in range(1, nf):
        if k + 1 < nf:
            submit(k + 1)
        l, t = ctx.kernel_launches(), time.perf_counter()
        if device_results:
            ctx.mseq_wait_device(out=out)
        else:
            ctx.mseq_wait()
        host += time.perf_counter() - t
        l_wait += ctx.kernel_launches() - l
        if device_results:              # the consumer: reads the poses and the inlier counts where they are
            acc += out["frame_pose"][:, :3, 3].sum() + out["counts"][:, 4].sum()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    steps = nf - 1
    return n * steps / dt, dt / steps, host / steps, l_sub / steps, l_wait / steps


def submit_host_cost(ctx, P_l, P_r, seqs, reps=50):
    """median host time of one vo_mseq_submit_device call [us]: through the binding, and the C call alone (descriptor
    tables built beforehand); each call is waited for outside the timed region"""
    n = len(seqs)
    ctx.mseq_begin_device([s[0][0] for s in seqs], [s[0][1] for s in seqs], P_l, P_r)
    lefts, rights = [s[1][0] for s in seqs], [s[1][1] for s in seqs]
    lt, rt, _ = ctx._device_pairs(lefts, rights, None, n, False)
    binding, call = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        ctx.mseq_submit_device(lefts, rights)
        binding.append(time.perf_counter() - t0)
        ctx.mseq_wait(want_points=False)
        t0 = time.perf_counter()
        rc = ctx.lib.vo_mseq_submit_device(ctx.h, lt, rt, 0, None)
        call.append(time.perf_counter() - t0)
        ctx._check(rc)
        ctx.mseq_wait(want_points=False)
    return 1e6 * float(np.median(binding)), 1e6 * float(np.median(call))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--counts", default="1,2,4,8,16,32")
    ap.add_argument("--mono-rotation", action="store_true", help="also time every mode with the mono_rotation branch")
    ap.add_argument("--mixed-calibration", action="store_true",
                    help="also time every vo_mseq_* count with a distinct calibration per sequence")
    ap.add_argument("--mixed-sizes", action="store_true",
                    help="also time every vo_mseq_* count with the KITTI training set's three image sizes")
    ap.add_argument("--device-input", action="store_true",
                    help="also time every vo_mseq_* count with frames resident in GPU memory (gray and BGR tensors)")
    ap.add_argument("--device-results", action="store_true",
                    help="also time device input with host waits against vo_mseq_wait_device (VO_MSEQ_DEVICE_RESULTS)")
    ap.add_argument("--mixed-params", action="store_true",
                    help="also time every vo_mseq_* count with one set of tracking parameters per sequence")
    ap.add_argument("--json", help="also write the result here")
    a = ap.parse_args()
    if a.mixed_sizes and a.counts == ap.get_default("counts"):
        a.counts = "3,11,32"
    if a.device_input and a.counts == ap.get_default("counts"):
        a.counts = "1,8,16,32"
    if (a.device_results or a.mixed_params) and a.counts == ap.get_default("counts"):
        a.counts = "1,8,32"
    counts = [int(c) for c in a.counts.split(",")]
    from visual_odom_b200 import capi, synth
    P_l, P_r = synth.proj_matrices()
    t0 = time.perf_counter()
    dr = drives(a.frames + 1)
    print(f"rendered {DRIVES} drives x {a.frames + 1} frames in {time.perf_counter() - t0:.0f} s", flush=True)
    monos = (False, True) if a.mono_rotation else (False,)
    mixes = (False, True) if a.mixed_calibration else (False,)
    modes = [(m, mono, mix) for m in ["seq"] + counts for mono in monos for mix in mixes if not (m == "seq" and mix)]
    if a.mixed_sizes:
        modes += [(m, mono, "sizes") for m in counts for mono in monos]
    if a.device_input:
        modes += [(m, False, kind) for m in counts for kind in ("dev-gray", "dev-bgr")]
    if a.device_results:
        modes += [(m, False, kind) for m in counts for kind in ("dres-host", "dres-dev")]
    if a.mixed_params:
        modes += [(m, False, "params") for m in counts]
    seqs = {n: [sequence(dr, q) for q in range(n)] for n in counts}
    mixed = {}
    if a.mixed_calibration:              # per count n: sequence q rendered with calibration(q, n), played like sequence(dr, q)
        t0 = time.perf_counter()
        for n in counts:
            cals = [calibration(q, n) for q in range(n)]
            md = drives(a.frames + 1, cals)
            mixed[n] = ([md[q] if (q // DRIVES) % 2 == 0 else md[q][::-1] for q in range(n)],
                        np.stack([synth.proj_matrices(c)[0] for c in cals]), np.stack([synth.proj_matrices(c)[1] for c in cals]))
        print(f"rendered the mixed-calibration sequences in {time.perf_counter() - t0:.0f} s", flush=True)
    sized = {}
    if a.mixed_sizes:                    # per count n: sequence q at KITTI_SIZES[q % 11], played like sequence(dr, q)
        t0 = time.perf_counter()
        by_size = {sz: (dr if sz == (W, H) else drives(a.frames + 1, size=sz)) for sz in set(KITTI_SIZES)}
        for n in counts:
            sized[n] = [sequence(by_size[KITTI_SIZES[q % len(KITTI_SIZES)]], q) for q in range(n)]
        print(f"rendered the drives at {len(by_size)} image sizes in {time.perf_counter() - t0:.0f} s", flush=True)
    dev = {}
    if a.device_input or a.device_results:  # every frame of every drive resident on the GPU, gray and BGR, before any timing
        import torch
        for kind in ("dev-gray", "dev-bgr") if a.device_input else ("dev-gray",):
            t = [[tuple(torch.from_numpy(np.ascontiguousarray(x if kind == "dev-gray" else np.repeat(x[:, :, None], 3, axis=2)))
                        .cuda() for x in pair) for pair in fr] for fr in dr]
            dev[kind] = {n: [sequence(t, q) for q in range(n)] for n in set(counts) | {32, 64}}
        torch.cuda.synchronize()
        print(f"resident on the GPU: {torch.cuda.memory_allocated() / 2**30:.2f} GiB", flush=True)
    ctx = capi.Context(0, max_features=4096)
    res = {m: dict(fps=[], lat=[], launches=[], host=[], wait_launches=[]) for m in modes}

    def run(mode, fr_cut=None):
        m, mono, mix = mode
        if m == "seq":
            fr = dr[0] if fr_cut is None else dr[0][:fr_cut]
            return run_seq(ctx, P_l, P_r, fr, mono)
        if mix in ("dres-host", "dres-dev"):
            s = dev["dev-gray"][m] if fr_cut is None else [x[:fr_cut] for x in dev["dev-gray"][m]]
            return run_mseq_dres(ctx, P_l, P_r, s, mix == "dres-dev")
        if mix in ("dev-gray", "dev-bgr"):
            s = dev[mix][m] if fr_cut is None else [x[:fr_cut] for x in dev[mix][m]]
            return run_mseq_device(ctx, P_l, P_r, s, "bgr" if mix == "dev-bgr" else None)
        if mix == "params":
            ctx.mseq_params(0, [PARAM_SETS[q % len(PARAM_SETS)] for q in range(m)])
            try:
                return run_mseq(ctx, P_l, P_r, seqs[m] if fr_cut is None else [x[:fr_cut] for x in seqs[m]], mono)
            finally:
                ctx.mseq_params(0, [None] * m)
        s, Pl, Pr = (sized[m], P_l, P_r) if mix == "sizes" else (mixed[m] if mix else (seqs[m], P_l, P_r))
        s = s if fr_cut is None else [x[:fr_cut] for x in s]
        return run_mseq(ctx, Pl, Pr, s, mono)

    for _ in range(a.rounds):
        for m in modes:
            run(m, 4)                     # warm-up: (re-)captures the mode's graphs, untimed
            r = run(m)
            fps, lat, launches = r[0], r[1], r[-2] if len(r) == 5 else r[2]
            res[m]["fps"].append(fps); res[m]["lat"].append(lat); res[m]["launches"].append(launches)
            if len(r) == 5:
                res[m]["host"].append(r[2]); res[m]["wait_launches"].append(r[4])
    host_cost = {n: submit_host_cost(ctx, P_l, P_r, dev["dev-gray"][n]) for n in (32, 64)} if a.device_input else {}
    ctx.close()
    out = dict(card=card(), image=f"{W}x{H}", frames=a.frames, rounds=a.rounds, in_flight=2, modes={})
    if host_cost:
        out["submit_device_host_us"] = {str(n): dict(binding=b, c_call=c) for n, (b, c) in host_cost.items()}
    print(f"card (name, power limit, max SM clock): {out['card']}")
    for mode in modes:
        r = res[mode]
        o = dict(aggregate_fps=float(np.median(r["fps"])), aggregate_fps_min=float(np.min(r["fps"])),
                 aggregate_fps_max=float(np.max(r["fps"])), step_latency_ms=1e3 * float(np.median(r["lat"])),
                 launches_per_submission=float(np.median(r["launches"])))
        if r["host"]:
            o.update(host_ms_per_step=1e3 * float(np.median(r["host"])), launches_per_wait=float(np.median(r["wait_launches"])))
        m, mono, mix = mode
        out["modes"][str(m) + ("+mono" if mono else "") + ("+sizes" if mix == "sizes" else f"+{mix}" if mix in ("dev-gray", "dev-bgr", "dres-host", "dres-dev", "params")
                               else "+mixed" if mix else "")] = o
        name = ("vo_seq (1 sequence)" if m == "seq" else f"vo_mseq n_seq = {m:2d}") + (", mono" if mono else "") + \
            (", KITTI sizes" if mix == "sizes" else ", device gray" if mix == "dev-gray" else ", device BGR" if mix == "dev-bgr"
             else ", dev in, host wait" if mix == "dres-host" else ", dev in, dev results" if mix == "dres-dev"
             else ", params per sequence" if mix == "params"
             else ", mixed cal." if mix else "")
        print(f"{name:40s}: {o['aggregate_fps']:8.0f} frames/s [{o['aggregate_fps_min']:.0f}, {o['aggregate_fps_max']:.0f}], "
              f"step {o['step_latency_ms']:.3f} ms, {o['launches_per_submission']:.1f} launches / submission"
              + (f", host {o['host_ms_per_step']:.3f} ms / step, {o['launches_per_wait']:.1f} launches / wait" if "host_ms_per_step" in o else ""))
    for n, (b, c) in host_cost.items():
        print(f"one vo_mseq_submit_device, n_seq = {n:2d}: host {b:.1f} us through the binding, {c:.1f} us in the C call")
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
