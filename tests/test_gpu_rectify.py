"""Rectification of raw stereo frames on the GPU (vo_remap, vo_seq_rectify, vo_mseq_rectify) against cv2 4.13:
vo_remap is cv2.remap(INTER_LINEAR, BORDER_CONSTANT 0) byte for byte at 1241 x 376 and at 3840 x 2160, and a sequence
run on raw frames with its rectification is, frame by frame, the same sequence run on the frames cv2 rectified on the
CPU (records, the four point lists, the carried FeatureSet and translation, frame_pose), from host gray and BGR, from
device gray / HWC / CHW, pushed and pipelined, graphs on and off.  In the multi-sequence mode plain and rectified slots of
different cameras and sizes mix, starts switch a slot between plain and rectified, and every sequence is what it gives
alone; launches per submission are the header's counts; every refusal leaves the run going on bit for bit."""
import os
import sys

import numpy as np
import pytest

from visual_odom_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rectify_ref as rr  # noqa: E402
from test_oracle_rectify import edge_maps  # noqa: E402

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
ARRAYS = ("rvec", "tvec", "R", "l0", "r0", "l1", "r1")
_mats = synth.rectify_cam_matrices
KITTI_RAW = synth.RECTIFY_CAMS["kitti_raw_left"]
# the rig of each size (cameras of synth.RECTIFY_CAMS)
RIGS = {(752, 480): ("euroc_cam0", "euroc_cam1"), (1241, 376): ("kitti_raw_left", "kitti_raw_right"),
        (640, 480): ("kitti_raw_right", "kitti_raw_left"), (700, 440): ("euroc_cam1", "euroc_cam0")}
N = 20


def rect_of(w, h):
    return synth.rectify_rig(*RIGS[(w, h)])


_DRIVES = {}


def drive(w, h, seed=3, n=N):
    """(P_l, P_r, raw gray frames, raw BGR frames, cv2-rectified gray frames): rendered frames pushed through the inverse
    distortion of the rig's cameras, and what cv2 makes of them (remap(cvtColor(raw)))."""
    key = (w, h, seed, n)
    if key not in _DRIVES:
        rect = rect_of(w, h)
        dist = {}
        for side in ("left", "right"):
            K, D, R, P = rect[side]
            # raw = rendered seen through the opposite lens: a strong, image-leaving distortion to undo
            dist[side] = cv2.initUndistortRectifyMap(K, -D, np.eye(3), K, (w, h), cv2.CV_32FC1)
        maps = {s: cv2.initUndistortRectifyMap(*rect[s][:3], rect[s][3][:, :3], (w, h), cv2.CV_32FC1) for s in rect}
        base = synth.stereo_unit(w, h, seed)
        rendered = [(base["l0"], base["r0"])]
        for k in range(1, n):
            u = synth.stereo_unit(w, h, seed, rvec=np.array((0.001, -0.003, 0.0005)) * k, tvec=np.array((0.01, -0.002, -0.2)) * k)
            rendered.append((u["l1"], u["r1"]))
        raw, bgr, want = [], [], []
        for pair in rendered:
            rp, bp, wp = [], [], []
            for side, img in zip(("left", "right"), pair):
                g = cv2.remap(img, *dist[side], cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT)
                c = np.ascontiguousarray(np.stack([g, np.roll(g, 1, axis=1), 255 - g], -1))     # a colour frame
                rp.append(g); bp.append(c)
                wp.append(cv2.remap(cv2.cvtColor(c, cv2.COLOR_BGR2GRAY), *maps[side], cv2.INTER_LINEAR,
                                    borderMode=cv2.BORDER_CONSTANT, borderValue=0))
            raw.append(tuple(rp)); bgr.append(tuple(bp)); want.append(tuple(wp))
        gray_want = [tuple(cv2.remap(g, *maps[s], cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT)
                           for s, g in zip(("left", "right"), p)) for p in raw]
        _DRIVES[key] = (base["P_l"], base["P_r"], raw, bgr, gray_want, want)
    return _DRIVES[key]


def same(a, b, where):
    for k in INTS:
        assert a[k] == b[k], f"{where}: {k} {a[k]} != {b[k]}"
    for k in ARRAYS:
        assert np.array_equal(np.asarray(a[k]).ravel(), np.asarray(b[k]).ravel()), f"{where}: {k}"
    if "mono" in a or "mono" in b:
        ma, mb = a["mono"], b["mono"]
        for k in ("status", "n_inliers", "ransac_iters", "n_good"):
            assert ma[k] == mb[k], f"{where}: mono {k}"
        assert np.array_equal(ma["R"], mb["R"]) and np.array_equal(ma["t"], mb["t"]), f"{where}: mono R / t"


def same_state(a, b, where):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y)), where


@pytest.mark.parametrize("w,h", [(1241, 376), (3840, 2160)])
def test_remap_is_cv2s(ctx, w, h):
    src = np.random.default_rng(w).integers(0, 256, (h, w), dtype=np.uint8)
    mx, my = edge_maps(w, h, 9)
    want = cv2.remap(src, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(ctx.remap(src, mx, my), want)
    K, D, R, P = _mats(KITTI_RAW)
    mx, my = cv2.initUndistortRectifyMap(K, D * 3, R, P[:, :3] * [[0.6], [0.6], [1]], (w, h), cv2.CV_32FC1)
    want = cv2.remap(src, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(ctx.remap(src, mx, my), want)
    assert np.array_equal(rr.remap(src, mx, my), want)


def run_seq(ctx, w, h, frames, kind="gray", rect=None, pipelined=False, device_order=None, mono=False):
    """vo_seq_* over the drive's frames: per frame (record, state, pose); mono: the option "mono_rotation" (gray push)."""
    P_l, P_r, raw, bgr, gray_want, want = drive(w, h)
    ctx.seq_rectify(rect)
    try:
        if mono:
            ctx.set_option("mono_rotation", 1)
            ctx.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
            return [(ctx.seq_push(l, r, mono=True), ctx.seq_state(), ctx.seq_pose()) for l, r in frames[1:]]
        if device_order:
            import torch
            def dev(a):
                t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
                return t.permute(2, 0, 1).contiguous() if device_order == "chw" else t
            order = None if device_order == "gray" else "bgr"
            ctx.seq_begin_device(dev(frames[0][0]), dev(frames[0][1]), P_l, P_r, order=order)
            out = [(ctx.seq_push_device(dev(l), dev(r), order=order), ctx.seq_state(), ctx.seq_pose()) for l, r in frames[1:]]
            return out
        if kind == "bgr":
            ctx.seq_begin_bgr(frames[0][0], frames[0][1], P_l, P_r)
            return [(ctx.seq_push_bgr(l, r), ctx.seq_state(), ctx.seq_pose()) for l, r in frames[1:]]
        ctx.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
        if not pipelined:
            return [(ctx.seq_push(l, r), ctx.seq_state(), ctx.seq_pose()) for l, r in frames[1:]]
        out = []
        ctx.seq_submit(*frames[1])
        for k in range(1, len(frames)):
            if k + 1 < len(frames):
                ctx.seq_submit(*frames[k + 1])
            out.append((ctx.seq_wait(), None, None))
        return out
    finally:
        ctx.seq_rectify(None)
        ctx.set_option("mono_rotation", 0)


def compare(a, b, what):
    assert len(a) == len(b)
    for k, ((ra, sa, pa), (rb, sb, pb)) in enumerate(zip(a, b)):
        same(ra, rb, f"{what} frame {k + 1}")
        if sa is not None and sb is not None:
            same_state(sa, sb, f"{what} frame {k + 1} state")
        if pa is not None and pb is not None:
            assert np.array_equal(pa, pb), f"{what} frame {k + 1} pose"
    assert sum(r["n_valid"] for r, _, _ in a) > 0, f"{what}: nothing was tracked"


@pytest.mark.parametrize("w,h", [(752, 480), (1241, 376)])
def test_sequence_on_raw_frames_is_the_sequence_on_cv2_rectified_frames(ctx, w, h):
    P_l, P_r, raw, bgr, gray_want, want = drive(w, h)
    rect = rect_of(w, h)
    ref = run_seq(ctx, w, h, gray_want)
    compare(run_seq(ctx, w, h, raw, rect=rect), ref, "host gray push")
    compare(run_seq(ctx, w, h, raw, rect=rect, pipelined=True), run_seq(ctx, w, h, gray_want, pipelined=True), "host gray pipelined")
    ctx.set_option("graphs", 0)
    try:
        compare(run_seq(ctx, w, h, raw, rect=rect), ref, "host gray, graphs off")
    finally:
        ctx.set_option("graphs", 1)
    ref_c = run_seq(ctx, w, h, want)
    compare(run_seq(ctx, w, h, bgr, kind="bgr", rect=rect), ref_c, "host BGR")
    compare(run_seq(ctx, w, h, raw, rect=rect, device_order="gray"), ref, "device gray")
    compare(run_seq(ctx, w, h, bgr, rect=rect, device_order="hwc"), ref_c, "device HWC")
    compare(run_seq(ctx, w, h, bgr, rect=rect, device_order="chw"), ref_c, "device CHW")


def test_cv2_rectified_run_closes_on_the_reference_glue(ctx):
    """The cv2-rectified frames run through the reference's glue (oracle/ref_path, cv2 backend) give the library's
    records on the first frames, so the chain raw -> rectified -> tracked ends at cv2."""
    from oracle import ref_path
    w, h = 752, 480
    P_l, P_r, raw, bgr, gray_want, want = drive(w, h)
    got = run_seq(ctx, w, h, raw, rect=rect_of(w, h))
    fs = ref_path.FeatureSet()
    for k in range(1, 4):
        (l0, r0), (l1, r1) = gray_want[k - 1], gray_want[k]
        pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend="cv2")
        r = got[k - 1][0]
        assert r["n_valid"] == len(pL0) > 0, f"frame {k}: {r['n_valid']} != {len(pL0)}"
        for name, pts in (("l0", pL0), ("r0", pR0), ("l1", pL1), ("r1", pR1)):
            assert np.array_equal(r[name], pts), f"frame {k}: {name}"
        pts, ages, _ = got[k - 1][1]
        assert np.array_equal(pts, fs.points) and np.array_equal(ages, fs.ages), f"frame {k}: carried FeatureSet"


def alone(ctx, w, h, rect, n, kind="gray", mono=False):
    P_l, P_r, raw, bgr, gray_want, want = drive(w, h)
    frames = (bgr if kind == "bgr" else raw)[:n]
    return run_seq(ctx, w, h, frames, kind=kind, rect=rect, mono=mono)


# (slot, first submission, size, rectified, frames).  Every start after the first submission changes its slot's size and
# comes in with host pairs (except in the device-results run): slot 1 goes from plain 640 x 480 to rectified 700 x 440,
# slot 0 from rectified 752 x 480 to rectified 640 x 480 (another rig), slot 2 from rectified 700 x 440 to plain 752 x 480.
MIXED = [(0, 1, (752, 480), True, 6), (1, 1, (640, 480), False, 4), (2, 2, (700, 440), True, 5),
         (1, 5, (700, 440), True, 6), (0, 7, (640, 480), True, 5), (2, 7, (752, 480), False, 5)]


def _dres_records(d, q):
    """seq_wait-style record of sequence q from the host copies of one mseq_wait_device result."""
    r = {f: int(d["counts"][q, i]) for i, f in enumerate(INTS)}
    r.update(rvec=d["rvec"][q], tvec=d["tvec"][q], R=d["R"][q], status=int(d["status"][q]))
    for i, f in enumerate(("l0", "r0", "l1", "r1")):
        r[f] = d["pts4"][q, i, :r["n_valid"]]
    return r


@pytest.mark.parametrize("kind", ["gray", "bgr", "mixed", "mono", "dres", "gray_pipelined", "bgr_pipelined"])
def test_multi_sequence_mixes_plain_and_rectified_slots_and_starts_switch_them(ctx, kind):
    """Plain and rectified slots of different rigs and sizes in one opened run, starts that switch a slot between plain
    and rectified and change its size: each sequence is, frame by frame, what it gives alone through vo_seq_* (records,
    point lists, carried state, frame_pose; with the mono flag the recoverPose results).  kind: every submission from host
    gray, from host BGR, host gray with every third submission from device memory, host gray with
    VO_MSEQ_MONO_ROTATION, or device input with VO_MSEQ_DEVICE_RESULTS (results through vo_mseq_wait_device).  The
    pipelined kinds keep two submissions in flight, so a start's pair is staged while the previous frame still runs (the
    geometry entries it is remapped at must be written before that staging); they check records and frame_pose."""
    import torch
    from visual_odom_b200.capi import VO_MSEQ_STARTED
    pipelined = kind.endswith("_pipelined")
    kind = kind.replace("_pipelined", "")
    mono, dres = kind == "mono", kind == "dres"
    K = max(k0 + L - 1 for _, k0, _, _, L in MIXED)
    ctx.mseq_open(3, 752, 480, mono_rotation=mono, device_results=dres)
    recs = {i: [] for i in range(len(MIXED))}
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def submit(k):
        lefts, rights, start = [None] * 3, [None] * 3, {}
        for i, (q, k0, (w, h), on, L) in enumerate(MIXED):
            if k0 <= k < k0 + L:
                P_l, P_r, raw, bgr, _, _ = drive(w, h)
                lefts[q], rights[q] = (bgr if kind == "bgr" else raw)[k - k0]
                if k == k0:
                    ctx.mseq_rectify(q, [rect_of(w, h) if on else None])
                    start[q] = (P_l, P_r)
        if dres or (kind == "mixed" and k % 3 == 0):
            order = "bgr" if kind == "bgr" else None
            ctx.mseq_submit_device([dev(a) for a in lefts], [dev(a) for a in rights], start=start, order=order)
        else:
            ctx.mseq_submit(lefts, rights, start=start)

    try:
        if pipelined:
            submit(1)
        for k in range(1, K + 1):
            if not pipelined:
                submit(k)
            elif k < K:
                submit(k + 1)
            if dres:
                got = ctx.mseq_wait_device()
                torch.cuda.synchronize()
                d = {f: v.cpu().numpy() for f, v in got.items() if isinstance(v, torch.Tensor)}
                out = [_dres_records(d, q) for q in range(3)]
            else:
                out = ctx.mseq_wait(mono=mono)
            for i, (q, k0, (w, h), on, L) in enumerate(MIXED):
                if k0 < k < k0 + L:
                    pose = ctx.mseq_pose(q)
                    if dres:
                        assert np.array_equal(d["frame_pose"][q], pose), f"sequence {i}: device frame_pose"
                    recs[i].append((out[q], None if pipelined else ctx.mseq_state(q), pose))
                elif k == k0:
                    assert out[q]["status"] == VO_MSEQ_STARTED
    finally:
        ctx.mseq_rectify(0, [None, None, None])
    for i, (q, k0, (w, h), on, L) in enumerate(MIXED):
        want = alone(ctx, w, h, rect_of(w, h) if on else None, L, kind="bgr" if kind == "bgr" else "gray", mono=mono)
        compare(recs[i], want, f"{kind}: slot {q} sequence {i}")


def _launches(ctx, n, rect_slots, device=False, bgr=False):
    """Launches of the third submission of an n-sequence vo_mseq_begin run whose slots rect_slots are rectified."""
    import torch
    w, h = 752, 480
    P_l, P_r, raw, bgrf, _, _ = drive(w, h)
    fr = bgrf if bgr else raw
    ctx.mseq_rectify(0, [rect_of(w, h) if q in rect_slots else None for q in range(n)])
    try:
        ctx.mseq_begin([fr[0][0]] * n, [fr[0][1]] * n, P_l, P_r)
        for k in (1, 2):
            ctx.mseq_submit([fr[k][0]] * n, [fr[k][1]] * n); ctx.mseq_wait(want_points=False)
        l0 = ctx.kernel_launches()
        if device:
            t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in fr[3]]
            ctx.mseq_submit_device([t[0]] * n, [t[1]] * n)
        else:
            ctx.mseq_submit([fr[3][0]] * n, [fr[3][1]] * n)
        ctx.mseq_wait(want_points=False)
        return ctx.kernel_launches() - l0
    finally:
        ctx.mseq_rectify(0, [None] * n)


@pytest.mark.parametrize("n", [1, 16])
def test_launch_counts_are_the_headers(ctx, n):
    some = {0} if n == 1 else {1, 5, 6, 15}
    assert _launches(ctx, n, some) == _launches(ctx, n, set()) + 1
    assert _launches(ctx, n, some, device=True) == _launches(ctx, n, set(), device=True)
    assert _launches(ctx, n, some, bgr=True) == _launches(ctx, n, set(), bgr=True)


def test_refusals_change_nothing(ctx):
    from visual_odom_b200.capi import VoError, VO_E_INVALID, rectify_struct
    w, h = 752, 480
    P_l, P_r, raw, _, gray_want, _ = drive(w, h)
    rect = rect_of(w, h)
    ref = run_seq(ctx, w, h, raw[:6], rect=rect)
    bad = []
    r = rectify_struct(rect); r.left.n_d = 6; bad.append(r)
    r = rectify_struct(rect); r.right.K[0] = float("nan"); bad.append(r)
    r = rectify_struct(rect); r.left.D[1] = float("inf"); bad.append(r)
    r = rectify_struct(rect); r.right.P[:] = [0.0] * 9; bad.append(r)
    r = rectify_struct(rect); r.left.R[:] = [1, 0, 0, 0, 0, 0, 0, 0, 1]; bad.append(r)
    ctx.seq_rectify(rect)
    P_l, P_r = drive(w, h)[:2]
    ctx.seq_begin(raw[0][0], raw[0][1], P_l, P_r)
    got = []
    for k in range(1, 6):
        for b in bad:
            with pytest.raises(VoError) as e:
                ctx.seq_rectify(b)
            assert e.value.code == VO_E_INVALID
            with pytest.raises(VoError) as e:
                ctx.mseq_rectify(k, [b])
            assert e.value.code == VO_E_INVALID
        with pytest.raises(VoError):
            ctx.mseq_rectify(63, [rect, rect])
        with pytest.raises(VoError):
            ctx.mseq_rectify(-1, [rect])
        got.append((ctx.seq_push(*raw[k]), ctx.seq_state(), ctx.seq_pose()))
    ctx.seq_rectify(None)
    compare(got, ref, "after refusals")
    # the refused calls left the setting as it was: a begin now runs rectified
    ctx.seq_rectify(rect)
    compare(run_seq(ctx, w, h, raw[:6], rect=rect), ref, "setting kept")


def test_retiring_the_last_rectified_sequence_restores_the_plain_launches(ctx):
    """Once the only rectified sequence has retired, a submission launches what the same run without rectification
    launches (host gray and host BGR, the latter back to its in-graph conversion)."""
    w, h = 752, 480
    P_l, P_r, raw, bgr, _, _ = drive(w, h)

    def counts(rect, colour):
        fr = bgr if colour else raw
        ctx.mseq_rectify(0, [None, rect_of(w, h) if rect else None])
        try:
            ctx.mseq_begin([fr[0][0]] * 2, [fr[0][1]] * 2, P_l, P_r)
            out = []
            for k in range(1, 7):
                l0 = ctx.kernel_launches()
                live = k < 3
                ctx.mseq_submit([fr[k][0], fr[k][0] if live else None], [fr[k][1], fr[k][1] if live else None])
                ctx.mseq_wait(want_points=False)
                out.append(ctx.kernel_launches() - l0)
            return out
        finally:
            ctx.mseq_rectify(0, [None, None])
    for colour in (False, True):
        plain, rect = counts(False, colour), counts(True, colour)
        assert rect[-2:] == plain[-2:], (colour, plain, rect)
        if not colour:
            assert rect[0] == plain[0] + 1, (plain, rect)
