#!/usr/bin/env python
"""The reference's `./run <dataset>/ <calibration.yaml>` (reference src/main.cpp:40-224) on the streaming sequence mode:

    python tools/run_sequence.py /data/kitti/sequences/00/ calibration/kitti00.yaml --poses out/00.txt [--gt poses/00.txt]

<dataset>/image_0/%06d.png and image_1/%06d.png are decoded ahead by the library's reader into pinned buffers, frames
are pushed through vo_seq_submit / vo_seq_wait (two in flight), frame_pose is integrated with the reference's Euler and
scale gates, the trajectory is written in the KITTI text format and, with --gt, scored with the KITTI segment metric.
`--mono-rotation` runs trackingFrame2Frame as its header default does (mono_rotation = true: the rotation from
findEssentialMat + recoverPose, the translation from the PnP; frames where that branch would abort are reported and not
integrated).  `--lk-win W` tracks with a W x W window (3 to 32; the reference's 21 by default).  `--rectify SETTINGS.yaml`
rectifies raw frames on the GPU as ORB-SLAM2's stereo driver does (initUndistortRectifyMap + remap(INTER_LINEAR) with the
settings file's LEFT / RIGHT K, D, R, P).  `--check` only validates the inputs (no GPU needed)."""
import argparse
import os
import re
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np


def read_calibration(path):
    """Camera.fx / fy / cx / cy / bf of the reference's OpenCV-YAML files (calibration/*.yaml; src/main.cpp:67-74)."""
    vals = {}
    for ln in open(path):
        m = re.match(r"\s*Camera\.(fx|fy|cx|cy|bf)\s*:\s*([-+0-9.eE]+)", ln)
        if m:
            vals[m.group(1)] = float(m.group(2))
    missing = [k for k in ("fx", "fy", "cx", "cy", "bf") if k not in vals]
    if missing:
        raise SystemExit(f"{path}: missing Camera.{missing[0]}")
    return vals


def _opencv_matrices(text):
    """name -> float64 array of every `name: !!opencv-matrix` node of an OpenCV-YAML text (rows, cols, data)."""
    out = {}
    for m in re.finditer(r"^\s*([\w.]+)\s*:\s*!!opencv-matrix\s*\n((?:[ \t]+.*\n?)+)", text, re.M):
        body = m.group(2)
        rows = int(re.search(r"rows\s*:\s*(\d+)", body).group(1))
        cols = int(re.search(r"cols\s*:\s*(\d+)", body).group(1))
        data = re.search(r"data\s*:\s*\[([^\]]*)\]", body, re.S).group(1)
        vals = np.array([float(v) for v in data.replace("\n", " ").split(",") if v.strip()], np.float64)
        if vals.size != rows * cols:
            raise SystemExit(f"{m.group(1)}: {vals.size} values for a {rows} x {cols} matrix")
        out[m.group(1)] = vals.reshape(rows, cols)
    return out


def read_rectify(path):
    """The rectification of an ORB-SLAM2 stereo settings file: {"left": (K, D, R, P), "right": (K, D, R, P),
    "size": (LEFT.width, LEFT.height)} from its LEFT.K / D / R / P and RIGHT.* opencv-matrix nodes (P is 3 x 4; the
    library takes its left 3 x 3).  What cv2.FileStorage reads from the same file, without cv2."""
    text = open(path).read()
    mats = _opencv_matrices(text)
    out = {}
    for side in ("LEFT", "RIGHT"):
        try:
            K, D, R, P = (mats[f"{side}.{k}"] for k in "KDRP")
        except KeyError as e:
            raise SystemExit(f"{path}: missing {e.args[0]}")
        if K.shape != (3, 3) or R.shape != (3, 3) or P.shape[0] != 3 or P.shape[1] not in (3, 4) or D.size not in (4, 5, 8):
            raise SystemExit(f"{path}: {side}: K, R must be 3 x 3, P 3 x 3 or 3 x 4, D 4, 5 or 8 coefficients")
        out[side.lower()] = (K, D.ravel(), R, P)
    size = [re.search(r"^\s*LEFT\.%s\s*:\s*(\d+)" % k, text, re.M) for k in ("width", "height")]
    out["size"] = tuple(int(m.group(1)) for m in size) if all(size) else None
    return out


def count_frames(dataset, first):
    n = 0
    while os.path.exists(os.path.join(dataset, "image_0", "%06d.png" % (first + n))) and \
            os.path.exists(os.path.join(dataset, "image_1", "%06d.png" % (first + n))):
        n += 1
    return n


def bucket_grid(w, h, divisor=10, per_bucket=1):
    """the points bucketingFeatures reads back at most: (rows/bs + 1) x (cols/bs + 1) cells of per_bucket slots,
    bs = rows / divisor (the library's seq_grid)"""
    bs = max(h // divisor, 1)
    return (h // bs + 1) * (w // bs + 1) * per_bucket


def add_bucket_args(ap):
    """matchingFeatures' bookkeeping (vo_params; the reference's literals by default)"""
    ap.add_argument("--features-per-bucket", type=int, default=1, help="Bucket(max_size) (default 1)")
    ap.add_argument("--bucket-divisor", type=int, default=10, help="bucket_size = rows / DIVISOR (default 10)")
    ap.add_argument("--age-threshold", type=int, default=10, help="buckets admit features aged < THRESHOLD (default 10)")
    ap.add_argument("--refill-threshold", type=int, default=2000,
                    help="FAST corners are appended while fewer than THRESHOLD features are tracked (default 2000)")


def add_lk_win_arg(ap):
    """calcOpticalFlowPyrLK's winSize (vo_params.lk_win): one value for the whole context"""
    ap.add_argument("--lk-win", type=int, default=21, metavar="W",
                    help="track with a W x W LK window, 3 <= W <= 32 (default 21, the reference's Size(21,21))")


def lk_win_param(a):
    if not 3 <= a.lk_win <= 32:
        raise SystemExit(f"--lk-win {a.lk_win}: the LK window runs from 3 to 32")
    return a.lk_win


def bucket_params(a, sizes):
    """the Context keywords of the flags; max_features is raised from 4096 to the largest read-back bound of the sizes"""
    if a.features_per_bucket < 1 or a.bucket_divisor < 1:
        raise SystemExit("--features-per-bucket and --bucket-divisor must be positive")
    for w, h in sizes:
        if h // a.bucket_divisor == 0:
            raise SystemExit(f"{w}x{h} images are too small for the rows/{a.bucket_divisor} bucket size")
    bound = max(bucket_grid(w, h, a.bucket_divisor, a.features_per_bucket) for w, h in sizes)
    return dict(max_features=max(4096, bound), refill_threshold=a.refill_threshold, bucket_rows_divisor=a.bucket_divisor,
                features_per_bucket=a.features_per_bucket, bucket_age_threshold=a.age_threshold)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("dataset"); ap.add_argument("calibration")
    ap.add_argument("--first", type=int, default=0); ap.add_argument("--frames", type=int, default=0, help="0 = all")
    ap.add_argument("--poses", help="write the trajectory here (KITTI format)")
    ap.add_argument("--gt", help="ground-truth poses to score against")
    ap.add_argument("--threads", type=int, default=8); ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--mono-rotation", action="store_true",
                    help="rotation from findEssentialMat + recoverPose (trackingFrame2Frame's header default)")
    add_bucket_args(ap)
    add_lk_win_arg(ap)
    ap.add_argument("--rectify", metavar="SETTINGS.yaml",
                    help="rectify the raw frames with the LEFT / RIGHT K, D, R, P of an ORB-SLAM2 stereo settings file")
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    from visual_odom_b200 import capi, synth
    cal = read_calibration(a.calibration)
    P_l, P_r = synth.proj_matrices(cal)
    n = count_frames(a.dataset, a.first)
    if a.frames:
        n = min(n, a.frames)
    if n < 2:
        raise SystemExit(f"{a.dataset}: need at least two stereo pairs (image_0/%06d.png, image_1/%06d.png from {a.first})")
    w, h, ctype, depth = capi.png_info(open(os.path.join(a.dataset, "image_0", "%06d.png" % a.first), "rb").read())
    print(f"{n} stereo pairs of {w}x{h} (PNG colour type {ctype}, {depth} bit); P_left =\n{P_l}\nP_right =\n{P_r}")
    print("rotation: " + ("findEssentialMat + recoverPose (mono_rotation = true)" if a.mono_rotation else
                          "Rodrigues of the PnP rvec (mono_rotation = false)"))
    rect = read_rectify(a.rectify) if a.rectify else None
    if rect:
        if rect["size"] and rect["size"] != (w, h):
            raise SystemExit(f"{a.rectify}: LEFT.width / height {rect['size']} differ from the {w}x{h} frames")
        print(f"rectification: {a.rectify} (initUndistortRectifyMap + remap(INTER_LINEAR) on the GPU)")
    prm = bucket_params(a, [(w, h)])
    prm["lk_win"] = lk_win_param(a)
    print(f"LK window: {a.lk_win}x{a.lk_win}")
    print(f"bucketing: {a.features_per_bucket} feature(s) per bucket of rows/{a.bucket_divisor}, ages < {a.age_threshold}, "
          f"refill below {a.refill_threshold} features; max_features {prm['max_features']}")
    if a.check:
        return
    ctx = capi.Context(a.device, max_units=2, **prm)
    ctx.set_option("mono_rotation", 1 if a.mono_rotation else 0)
    ctx.seq_rectify(rect)
    aborted = 0
    rd = capi.SequenceReader(a.dataset, a.first, n, threads=a.threads, depth=a.threads + 3)
    lp, rp, rw, rh, pitch, ch, fid = rd.next_ptr()
    ctx.seq_begin_ptr(rw, rh, lp, rp, pitch, P_l, P_r, ch)
    poses = [np.eye(4)]
    t0 = time.perf_counter()
    lp, rp, rw, rh, pitch, ch, fid = rd.next_ptr()
    ctx.seq_submit_ptr(lp, rp, pitch, ch)
    for k in range(1, n):
        if k + 1 < n:
            lp, rp, rw, rh, pitch, ch, fid = rd.next_ptr()
            ctx.seq_submit_ptr(lp, rp, pitch, ch)
        res = ctx.seq_wait(want_points=False, mono=a.mono_rotation)
        if a.mono_rotation and res["mono"]["status"] != capi.VO_OK:
            aborted += 1
        poses.append(ctx.seq_pose())
        if k % 100 == 0 or k == n - 1:
            dt = time.perf_counter() - t0
            print(f"frame {a.first + k}: {res['n_valid']} matches, {res['n_inliers']} inliers, "
                  f"position {poses[-1][:3, 3].round(2)}, {k / dt:.0f} frames/s")
    rd.close(); ctx.close()
    if a.mono_rotation:
        print(f"{aborted} frames where findEssentialMat / recoverPose would abort (reported, not integrated)")
    if a.poses:
        os.makedirs(os.path.dirname(os.path.abspath(a.poses)), exist_ok=True)
        capi.poses_save(a.poses, poses)
    if a.gt:
        gt = capi.poses_load(a.gt)[a.first:a.first + n]
        seg, t_err, r_err = capi.eval_segments(gt, poses[:len(gt)])
        if len(seg) == 0:
            print("KITTI metric: the ground-truth path is shorter than the 100 m minimum segment, nothing to score")
        else:
            print(f"KITTI metric over {len(seg)} segments: t_err {100 * t_err:.2f} %, r_err {r_err * 180 / np.pi * 100:.4f} deg / 100 m")


if __name__ == "__main__":
    main()
