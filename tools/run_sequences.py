#!/usr/bin/env python
"""Several KITTI sequences through ONE context (the multi-sequence mode, vo_mseq_*), each with its own calibration:

    python tools/run_sequences.py /data/kitti/sequences/00/ /data/kitti/sequences/04/ calibration/kitti00.yaml \\
        --calibration-for 04=calibration/kitti04.yaml --poses out/ [--gt /data/kitti/poses/]

Every <dataset>/image_0/%06d.png and image_1/%06d.png is decoded ahead by its own library reader into pinned buffers; one
submission advances every sequence by one frame (two submissions in flight), and a sequence is retired at its last
frame, so sequences of unequal length share the run.  frame_pose of each is integrated with the reference's Euler and
scale gates (src/main.cpp:196-208), written to OUTDIR/<name>.txt in the KITTI text format (<name> = the dataset
directory's name) and, with --gt, scored against GTDIR/<name>.txt with the KITTI segment metric.  All sequences must
have the image size of the first, unless `--mixed-sizes` runs each at its own size (vo_mseq_begin_sized: KITTI's
training sequences come in three sizes, 1241x376, 1242x375 and 1226x370), which needs one pyramid depth for all of them
(every size above about 170 pixels on each side has the full depth).  The positional calibration applies to every sequence that no
`--calibration-for NAME=YAML` names (NAME = the dataset directory's name); each sequence runs with the matrices built from
its own file, as the reference's main() builds them (src/main.cpp:67-74).  `--mono-rotation` runs trackingFrame2Frame
as its header default does, for every sequence (mono_rotation = true: the rotation from findEssentialMat + recoverPose,
the translation from the PnP; frames where that branch would abort are reported and not integrated).  `--slots N` runs
the datasets as a queue through N slots (vo_mseq_open + vo_mseq_submit_start): the first N start together, and each
next one starts in the first slot that frees (the lowest slot on a tie), in the order given, so any number of datasets
runs through one context; their sizes may differ (one pyramid depth, the envelope of all of them), and every pose file
is the same for every N.  `--params-for NAME=FIELD=V[,FIELD=V...]` gives the dataset NAME its own tracking parameters
(vo_params fields such as fast_threshold, lk_max_iters, circ_threshold, pnp_reproj_error or features_per_bucket; the
context-wide lk_win, lk_max_level, fast_nonmax, max_features and max_units are refused); each sequence runs in its own
slot as a context created with its parameters would run it alone (vo_mseq_params).  `--sweep FIELD=V1,V2,...` runs the
first dataset once per value, each in its own slot of one context, with pose files OUTDIR/<name>_<FIELD>=<V>.txt.
`--lk-win W` tracks every sequence with a W x W LK window (3 to 32; the reference's 21 by default; one window per
context, so a dataset's --params-for cannot set it).  `--check` only validates the inputs and prints each sequence's parameters and the schedule of --slots (no GPU needed)."""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np

from run_sequence import (add_bucket_args, add_lk_win_arg, bucket_grid, bucket_params, count_frames, lk_win_param,
                          read_calibration, read_rectify)


def pyramid_depth(w, h, win):
    """pyramid images of a w x h image as the library builds them (vo_pyr_depth, csrc/common.cuh): levels up to the
    default vo_params.lk_max_level (read from the library's vo_default_params, which the run's context is created with),
    a level dropped once it is not larger than the win x win window (--lk-win)."""
    import ctypes as C
    from visual_odom_b200 import capi
    p = capi.VoParams()
    capi.load_library().vo_default_params(C.byref(p))
    n = 1
    for _ in range(p.lk_max_level):
        w, h = (w + 1) // 2, (h + 1) // 2
        if w <= win or h <= win:
            break
        n += 1
    return n


# vo_params fields a slot may set (vo_mseq_params); the others are the context's
SEQ_FIELDS = ("fast_threshold", "lk_max_iters", "lk_epsilon", "lk_min_eig", "circ_threshold", "pnp_iterations",
              "pnp_reproj_error", "pnp_confidence", "refill_threshold", "bucket_rows_divisor", "features_per_bucket",
              "bucket_age_threshold")


def parse_fields(spec, what):
    """FIELD=V[,FIELD=V...] -> {field: value} typed as vo_params declares the field"""
    import ctypes as C
    from visual_odom_b200 import capi
    types = dict(capi.VoParams._fields_)
    out = {}
    for item in spec.split(","):
        field, sep, v = item.partition("=")
        if not sep or not field or not v:
            raise SystemExit(f"{what} {spec}: expected FIELD=VALUE[,FIELD=VALUE...]")
        if field not in types:
            raise SystemExit(f"{what} {spec}: vo_params has no field {field}")
        if field not in SEQ_FIELDS:
            raise SystemExit(f"{what} {spec}: {field} is context-wide (one value for every sequence of a context)")
        try:
            out[field] = int(v) if types[field] is C.c_int else float(v)
        except ValueError:
            raise SystemExit(f"{what} {spec}: {field} takes {'an integer' if types[field] is C.c_int else 'a number'}, not {v}")
    return out


def queue_schedule(lengths, n_slots):
    """(slot, first submission) of each sequence of the given lengths (frames) run as a queue through n_slots slots: a
    sequence occupies its slot from the submission of its first pair to that of its last, and the next one starts in the
    first slot that frees (lowest index on a tie) at the submission after."""
    free_at = [1] * n_slots
    out = []
    for n in lengths:
        q = min(range(n_slots), key=lambda s: (free_at[s], s))
        out.append((q, free_at[q]))
        free_at[q] += n
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("datasets", nargs="+", metavar="DIR")
    ap.add_argument("calibration")
    ap.add_argument("--poses", required=True, metavar="OUTDIR", help="write OUTDIR/<name>.txt per sequence (KITTI format)")
    ap.add_argument("--gt", metavar="GTDIR", help="score each sequence against GTDIR/<name>.txt")
    ap.add_argument("--threads", type=int, default=4, help="decoder threads per sequence")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--mono-rotation", action="store_true",
                    help="rotation from findEssentialMat + recoverPose (trackingFrame2Frame's header default)")
    ap.add_argument("--calibration-for", action="append", default=[], metavar="NAME=YAML",
                    help="calibration of the dataset named NAME (repeatable; the others use the positional one)")
    ap.add_argument("--rectify-for", action="append", default=[], metavar="NAME=SETTINGS.yaml",
                    help="rectify the raw frames of the dataset named NAME with the LEFT / RIGHT K, D, R, P of an "
                         "ORB-SLAM2 stereo settings file (repeatable; the others run as they are)")
    ap.add_argument("--mixed-sizes", action="store_true",
                    help="run sequences of different image sizes together, each at its own size")
    ap.add_argument("--slots", type=int, metavar="N",
                    help="run the datasets as a queue through N slots, each starting in the first slot that frees")
    add_bucket_args(ap)
    add_lk_win_arg(ap)
    ap.add_argument("--params-for", action="append", default=[], metavar="NAME=FIELD=V[,FIELD=V...]",
                    help="tracking parameters of the dataset named NAME (repeatable; the others use the flags' values)")
    ap.add_argument("--sweep", metavar="FIELD=V1,V2,...",
                    help="run the first dataset once per value of FIELD, each in its own slot of one context")
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    from visual_odom_b200 import capi, synth
    default_cal = read_calibration(a.calibration)
    lk_win_param(a)
    if a.slots is not None and not 1 <= a.slots <= capi.VO_MSEQ_MAX:
        raise SystemExit(f"--slots {a.slots}: one context holds 1 to {capi.VO_MSEQ_MAX} slots")
    sized = a.mixed_sizes or a.slots is not None
    if a.slots is None and len(a.datasets) > capi.VO_MSEQ_MAX:
        raise SystemExit(f"{len(a.datasets)} sequences: one context runs at most {capi.VO_MSEQ_MAX}")
    names = [os.path.basename(os.path.normpath(d)) for d in a.datasets]
    if len(set(names)) != len(names):
        raise SystemExit(f"two datasets share a directory name ({names}): their pose files would collide")
    params_for = {}
    for spec in a.params_for:
        name, sep, rest = spec.partition("=")
        if not sep or not name:
            raise SystemExit(f"--params-for {spec}: expected NAME=FIELD=VALUE[,FIELD=VALUE...]")
        if name not in names:
            raise SystemExit(f"--params-for {spec}: no dataset is named {name} (names: {', '.join(names)})")
        if name in params_for:
            raise SystemExit(f"--params-for: {name} is given twice")
        params_for[name] = parse_fields(rest, "--params-for")
    sweep = None
    if a.sweep:
        field, sep, values = a.sweep.partition("=")
        if a.slots is not None:
            raise SystemExit("--sweep runs every value in a slot of its own: it does not combine with --slots")
        sweep = [(v, parse_fields(f"{field}={v}", "--sweep")) for v in values.split(",")] if sep else None
        if not sweep or len(sweep) > capi.VO_MSEQ_MAX or len({v for v, _ in sweep}) != len(sweep):
            raise SystemExit(f"--sweep {a.sweep}: expected FIELD=V1,V2,... with 1 to {capi.VO_MSEQ_MAX} distinct values")
    cal_for = {}
    for spec in a.calibration_for:
        name, sep, path = spec.partition("=")
        if not sep or not name or not path:
            raise SystemExit(f"--calibration-for {spec}: expected NAME=YAML")
        if name not in names:
            raise SystemExit(f"--calibration-for {spec}: no dataset is named {name} (names: {', '.join(names)})")
        if name in cal_for:
            raise SystemExit(f"--calibration-for: {name} is given twice")
        if not os.path.isfile(path):
            raise SystemExit(f"--calibration-for {spec}: {path} does not exist")
        cal_for[name] = (path, read_calibration(path))
    rect_for = {}
    for spec in a.rectify_for:
        name, sep, path = spec.partition("=")
        if not sep or not name or not path:
            raise SystemExit(f"--rectify-for {spec}: expected NAME=SETTINGS.yaml")
        if name not in names:
            raise SystemExit(f"--rectify-for {spec}: no dataset is named {name} (names: {', '.join(names)})")
        if name in rect_for:
            raise SystemExit(f"--rectify-for: {name} is given twice")
        if not os.path.isfile(path):
            raise SystemExit(f"--rectify-for {spec}: {path} does not exist")
        rect_for[name] = (path, read_rectify(path))
    seqs = []
    for d, name in zip(a.datasets, names):
        n = count_frames(d, 0)
        if n < 2:
            raise SystemExit(f"{d}: need at least two stereo pairs (image_0/%06d.png, image_1/%06d.png from 0)")
        w, h, ctype, depth = capi.png_info(open(os.path.join(d, "image_0", "%06d.png" % 0), "rb").read())
        if seqs and (w, h) != (seqs[0]["w"], seqs[0]["h"]) and not sized:
            raise SystemExit(f"{d}: {w}x{h} images, {a.datasets[0]} has {seqs[0]['w']}x{seqs[0]['h']}: "
                             "one context runs one image size (group the sequences by size, or run them together with "
                             "--mixed-sizes)")
        if sized and h // max(a.bucket_divisor, 1) == 0:
            raise SystemExit(f"{d}: {w}x{h} images are too small for the rows/{a.bucket_divisor} bucket size")
        if sized and seqs and pyramid_depth(w, h, a.lk_win) != pyramid_depth(seqs[0]["w"], seqs[0]["h"], a.lk_win):
            raise SystemExit(f"{d}: {w}x{h} images have {pyramid_depth(w, h, a.lk_win)} pyramid levels, {a.datasets[0]} "
                             f"({seqs[0]['w']}x{seqs[0]['h']}) has {pyramid_depth(seqs[0]['w'], seqs[0]['h'], a.lk_win)}: "
                             "one context runs one pyramid depth")
        gt = os.path.join(a.gt, name + ".txt") if a.gt else None
        if gt and not os.path.exists(gt):
            raise SystemExit(f"{gt}: no ground truth for sequence {name}")
        cal_path, cal = cal_for.get(name, (a.calibration, default_cal))
        P_l, P_r = synth.proj_matrices(cal)
        rect_path, rect = rect_for.get(name, (None, None))
        if rect and rect["size"] and rect["size"] != (w, h):
            raise SystemExit(f"{rect_path}: LEFT.width / height {rect['size']} differ from {name}'s {w}x{h} frames")
        seqs.append(dict(dir=d, name=name, n=n, w=w, h=h, gray=ctype == 0, gt=gt, P_l=P_l, P_r=P_r, own=params_for.get(name, {}),
                         rect=rect))
        print(f"{name}: {n} stereo pairs of {w}x{h} (PNG colour type {ctype}, {depth} bit), calibration {cal_path}"
              + (f", rectified with {rect_path}" if rect else ""))
        print(f"  P_left =\n{P_l}\n  P_right =\n{P_r}")
        if sweep:
            break                            # the sweep runs the first dataset only
    if sweep:
        first = seqs.pop()
        field = a.sweep.partition("=")[0]
        for v, own in sweep:
            seqs.append(dict(first, name=f"{first['name']}_{field}={v}", own=dict(first["own"], **own)))
    # each sequence's parameters: the flags' values (the library's defaults elsewhere), then its own
    import ctypes as C
    base = capi.VoParams()
    capi.load_library().vo_default_params(C.byref(base))
    flags = dict(refill_threshold=a.refill_threshold, bucket_rows_divisor=a.bucket_divisor,
                 features_per_bucket=a.features_per_bucket, bucket_age_threshold=a.age_threshold)
    for s in seqs:
        s["params"] = {f: flags.get(f, getattr(base, f)) for f in SEQ_FIELDS}
        s["params"].update(s["own"])
        p = s["params"]
        if p["features_per_bucket"] < 1 or p["bucket_rows_divisor"] < 1:
            raise SystemExit(f"{s['name']}: features_per_bucket and bucket_rows_divisor must be positive")
        if s["h"] // p["bucket_rows_divisor"] == 0:
            raise SystemExit(f"{s['name']}: {s['w']}x{s['h']} images are too small for the rows/{p['bucket_rows_divisor']} bucket size")
        s["grid"] = bucket_grid(s["w"], s["h"], p["bucket_rows_divisor"], p["features_per_bucket"])
    if sweep or params_for:
        for s in seqs:
            print(f"{s['name']}: " + " ".join(f"{f}={s['params'][f]:g}" for f in SEQ_FIELDS))
    if sized:
        print("image sizes: " + ", ".join(f"{s['name']} {s['w']}x{s['h']}" for s in seqs))
    if a.slots is not None:
        W, H = max(s["w"] for s in seqs), max(s["h"] for s in seqs)
        if pyramid_depth(W, H, a.lk_win) != pyramid_depth(seqs[0]["w"], seqs[0]["h"], a.lk_win):
            raise SystemExit(f"the envelope {W}x{H} of the sizes has {pyramid_depth(W, H, a.lk_win)} pyramid levels, the sizes "
                             f"{pyramid_depth(seqs[0]['w'], seqs[0]['h'], a.lk_win)}: one context runs one pyramid depth")
        # every slot opens at the densest sequence's parameters, which size the mono scratch for the envelope
        densest = max(seqs, key=lambda s: bucket_grid(W, H, s["params"]["bucket_rows_divisor"], s["params"]["features_per_bucket"]))
        a.open_params = densest["params"]
        env = bucket_grid(W, H, a.open_params["bucket_rows_divisor"], a.open_params["features_per_bucket"])
        for s in seqs:
            if a.mono_rotation and s["grid"] > env:
                raise SystemExit(f"{s['dir']}: {s['w']}x{s['h']} reads back {s['grid']} points, more than "
                                 f"the {env} of the envelope {W}x{H} the mono scratch is sized for")
        sched = queue_schedule([s["n"] for s in seqs], a.slots)
        steps = max(k0 + s["n"] - 1 for s, (_, k0) in zip(seqs, sched))
        print(f"schedule: {len(seqs)} sequences through {a.slots} slots of {W}x{H}, {steps} submissions")
        for s, (q, k0) in zip(seqs, sched):
            s["slot"], s["k0"] = q, k0
            print(f"  {s['name']}: slot {q}, submissions {k0}..{k0 + s['n'] - 1}")
    print("rotation: " + ("findEssentialMat + recoverPose (mono_rotation = true)" if a.mono_rotation else
                          "Rodrigues of the PnP rvec (mono_rotation = false)"))
    prm = bucket_params(a, [(s["w"], s["h"]) for s in seqs] + ([(W, H)] if a.slots is not None else []))
    # max_features covers every sequence's own bound, and pnp_iterations (the RANSAC scratch) every sequence's count;
    # each sequence then runs with its own parameters
    prm["max_features"] = max([prm["max_features"]] + [s["grid"] for s in seqs] +
                              ([env] if a.slots is not None else []))
    prm["pnp_iterations"] = max(max(s["params"]["pnp_iterations"] for s in seqs), base.pnp_iterations)
    prm["lk_win"] = a.lk_win
    print(f"LK window: {a.lk_win}x{a.lk_win} (every sequence)")
    print(f"bucketing: {a.features_per_bucket} feature(s) per bucket of rows/{a.bucket_divisor}, ages < {a.age_threshold}, "
          f"refill below {a.refill_threshold} features; max_features {prm['max_features']}")
    if a.check:
        return
    a.context_params = prm
    if a.slots is not None:
        return run_queue(a, capi, seqs, sched, W, H)
    # one pitch and one channel count per submission: colour files are read as BGR (converted on the device) unless the
    # sequences mix gray and colour files, then all are converted to gray while decoding
    force = 0 if len({s["gray"] for s in seqs}) == 1 else 1
    ctx = capi.Context(a.device, **a.context_params)
    ctx.mseq_params(0, [s["params"] for s in seqs])
    ctx.mseq_rectify(0, [s["rect"] for s in seqs])
    rds = [capi.SequenceReader(s["dir"], 0, s["n"], threads=a.threads, depth=a.threads + 3, force_channels=force) for s in seqs]

    def pairs(k):
        """pointers of frame k of every sequence (None past a sequence's last frame), pitch (one per sequence with
        --mixed-sizes: its reader's), channels"""
        lp, rp, fmt, pitches, chs = [], [], set(), [], set()
        for s, rd in zip(seqs, rds):
            if k >= s["n"]:
                lp.append(None); rp.append(None); pitches.append(s["w"])
                continue
            l, r, _, _, pitch, ch, _ = rd.next_ptr()
            lp.append(l); rp.append(r); fmt.add((pitch, ch)); pitches.append(pitch); chs.add(ch)
        if len(chs) > 1 or (len(fmt) > 1 and not a.mixed_sizes):
            raise SystemExit(f"frame {k}: the readers deliver different layouts {sorted(fmt)}")
        ch = chs.pop() if chs else 1
        if a.mixed_sizes:
            return lp, rp, pitches, ch
        pitch = fmt.pop()[0] if fmt else seqs[0]["w"]
        return lp, rp, pitch, ch

    lp, rp, pitch, ch = pairs(0)
    P_l = np.stack([s["P_l"] for s in seqs]); P_r = np.stack([s["P_r"] for s in seqs])
    if a.mixed_sizes:
        ctx.mseq_begin_ptr([s["w"] for s in seqs], [s["h"] for s in seqs], lp, rp, pitch, P_l, P_r, ch,
                           mono_rotation=a.mono_rotation)
    else:
        ctx.mseq_begin_ptr(seqs[0]["w"], seqs[0]["h"], lp, rp, pitch, P_l, P_r, ch, mono_rotation=a.mono_rotation)
    poses = [[np.eye(4)] for _ in seqs]
    aborted = [0] * len(seqs)
    steps = max(s["n"] for s in seqs)
    t0 = time.perf_counter()
    done = 0
    ctx.mseq_submit_ptr(*pairs(1))
    for k in range(1, steps):
        if k + 1 < steps:
            ctx.mseq_submit_ptr(*pairs(k + 1))
        recs = ctx.mseq_wait(want_points=False, mono=a.mono_rotation)
        for q, r in enumerate(recs):
            if r["status"] == capi.VO_MSEQ_RETIRED:
                continue
            if r["status"] != capi.VO_OK:
                print(f"{seqs[q]['name']} frame {k}: status {r['status']} ({ctx.lib.vo_last_error(ctx.h).decode()})")
            if a.mono_rotation and r["mono"]["status"] != capi.VO_OK:
                aborted[q] += 1
            poses[q].append(ctx.mseq_pose(q))
            done += 1
        if k % 100 == 0 or k == steps - 1:
            print(f"step {k}: {done} sequence-frames, {done / (time.perf_counter() - t0):.0f} frames/s")
    for rd in rds:
        rd.close()
    ctx.close()
    os.makedirs(a.poses, exist_ok=True)
    for s, p, n_abort in zip(seqs, poses, aborted):
        path = os.path.join(a.poses, s["name"] + ".txt")
        capi.poses_save(path, p)
        line = f"{s['name']}: {len(p)} poses -> {path}"
        if a.mono_rotation:
            line += f", {n_abort} frames where findEssentialMat / recoverPose would abort (reported, not integrated)"
        if s["gt"]:
            gt = capi.poses_load(s["gt"])[:len(p)]
            seg, t_err, r_err = capi.eval_segments(gt, p[:len(gt)])
            line += (", ground-truth path shorter than the 100 m minimum segment" if len(seg) == 0 else
                     f", KITTI metric over {len(seg)} segments: t_err {100 * t_err:.2f} %, r_err {r_err * 180 / np.pi * 100:.4f} deg / 100 m")
        print(line)


def run_queue(a, capi, seqs, sched, W, H):
    """--slots: every dataset starts in its scheduled slot (vo_mseq_submit_start) and retires after its last frame."""
    force = 0 if len({s["gray"] for s in seqs}) == 1 else 1
    ctx = capi.Context(a.device, **a.context_params)
    ctx.mseq_params(0, [a.open_params] * a.slots)
    ctx.mseq_open(a.slots, W, H, mono_rotation=a.mono_rotation)
    steps = max(s["k0"] + s["n"] - 1 for s in seqs)
    rds = {}                   # dataset index -> its reader, opened at its first pair, closed after its last wait
    by_step = {}
    for i, s in enumerate(seqs):
        for k in range(s["k0"], s["k0"] + s["n"]):
            by_step.setdefault(k, []).append(i)

    def submit(k):
        lp, rp, pitches, chs, start = [None] * a.slots, [None] * a.slots, [0] * a.slots, set(), {}
        for i in by_step.get(k, []):
            s = seqs[i]
            if k == s["k0"]:
                rds[i] = capi.SequenceReader(s["dir"], 0, s["n"], threads=a.threads, depth=a.threads + 3, force_channels=force)
                start[s["slot"]] = (s["w"], s["h"], s["P_l"], s["P_r"])
                ctx.mseq_params(s["slot"], [s["params"]])         # read by the start (host state: the slot may be in flight)
                ctx.mseq_rectify(s["slot"], [s["rect"]])
            l, r, _, _, pitch, ch, _ = rds[i].next_ptr()
            lp[s["slot"]], rp[s["slot"]], pitches[s["slot"]] = l, r, pitch
            chs.add(ch)
        if len(chs) > 1:
            raise SystemExit(f"submission {k}: the readers deliver different channel counts {sorted(chs)}")
        ctx.mseq_submit_ptr(lp, rp, pitches, chs.pop() if chs else 1, start=start)

    poses = [[np.eye(4)] for _ in seqs]
    aborted = [0] * len(seqs)
    t0 = time.perf_counter()
    done = 0
    submit(1)
    for k in range(1, steps + 1):
        if k + 1 <= steps:
            submit(k + 1)
        recs = ctx.mseq_wait(want_points=False, mono=a.mono_rotation)
        for i in by_step.get(k, []):
            s = seqs[i]
            r = recs[s["slot"]]
            if k == s["k0"]:
                continue                     # VO_MSEQ_STARTED: the first pair
            if r["status"] != capi.VO_OK:
                print(f"{s['name']} frame {k - s['k0']}: status {r['status']} ({ctx.lib.vo_last_error(ctx.h).decode()})")
            if a.mono_rotation and r["mono"]["status"] != capi.VO_OK:
                aborted[i] += 1
            poses[i].append(ctx.mseq_pose(s["slot"]))
            done += 1
            if k == s["k0"] + s["n"] - 1:
                rds.pop(i).close()           # its last submission has been waited for
        if k % 100 == 0 or k == steps:
            print(f"step {k}: {done} sequence-frames, {done / (time.perf_counter() - t0):.0f} frames/s")
    ctx.close()
    os.makedirs(a.poses, exist_ok=True)
    for s, p, n_abort in zip(seqs, poses, aborted):
        path = os.path.join(a.poses, s["name"] + ".txt")
        capi.poses_save(path, p)
        line = f"{s['name']}: {len(p)} poses -> {path}"
        if a.mono_rotation:
            line += f", {n_abort} frames where findEssentialMat / recoverPose would abort (reported, not integrated)"
        if s["gt"]:
            gt = capi.poses_load(s["gt"])[:len(p)]
            seg, t_err, r_err = capi.eval_segments(gt, p[:len(gt)])
            line += (", ground-truth path shorter than the 100 m minimum segment" if len(seg) == 0 else
                     f", KITTI metric over {len(seg)} segments: t_err {100 * t_err:.2f} %, r_err {r_err * 180 / np.pi * 100:.4f} deg / 100 m")
        print(line)


if __name__ == "__main__":
    main()
