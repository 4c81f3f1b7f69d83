"""Sequences started in free slots of a running multi-sequence context (vo_mseq_open / vo_mseq_submit_start): every
started sequence is, frame by frame, what vo_seq_begin(first pair) + vo_seq_push give on a fresh context (records, the
four point lists, the carried FeatureSet and translation, frame_pose, and with VO_MSEQ_MONO_ROTATION the mono results and
essential masks).  Every sequence of a run is checked this way, so the bystanders of a start are checked against what
they give with no start at all.  The cases: starts into empty slots, into a slot retired long before, into the slot that
the submission in flight retires, in place of a live sequence with another calibration (two in flight), after a larger
image, with a larger bucket grid, the mono branch, colour input, graphs off, pipelining, several starts at once, a queue
of drives through three slots, launch counts, one started sequence against cv2, and every refusal."""
import ctypes as C

import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

K0 = synth.KITTI00
NMAX = 6                    # frames per drive at most
ENV = (656, 248)            # the envelope of the opened runs


def _cal(sx=1.0, sy=1.0, dcx=0.0, dcy=0.0, sb=1.0):
    return dict(fx=K0["fx"] * sx, fy=K0["fy"] * sy, cx=K0["cx"] + dcx, cy=K0["cy"] + dcy, bf=K0["bf"] * sb)


# (w, h, seed, per-frame rotation, per-frame translation, calibration); 3 pans right and down, 4 has a larger bucket grid
# than the envelope (656 x 200: 363 cells against 308)
DRIVES = [
    (640, 240, 31, (0.001, -0.004, 0.0005), (0.01, -0.003, -0.2), _cal()),
    (601, 233, 7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25), _cal(0.9, 0.9, -300.0, -60.0)),
    (656, 248, 13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15), _cal(1.1, 1.1, -280.0, -55.0)),
    (512, 200, 42, (-0.006, 0.012, 0.0005), (0.03, 0.01, -0.3), _cal(1.0, 1.0, -350.0, -85.0, 1.15)),
    (656, 200, 13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15), _cal(1.1, 1.1, -280.0, -85.0)),
    (512, 248, 42, (0.001, -0.003, 0.0005), (0.01, 0.0, -0.2), _cal(1.0, 1.0, -350.0, -60.0)),
    (640, 240, 5, (0.002, 0.001, 0.0), (0.0, 0.002, -0.22), _cal(0.95, 0.95, -10.0, 5.0, 0.9)),
    (620, 236, 23, (-0.001, -0.002, 0.0005), (0.01, 0.0, -0.18), _cal(1.05, 1.05, -290.0, -70.0)),
]
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
ARRAYS = ("rvec", "tvec", "R", "l0", "r0", "l1", "r1")

_FRAMES = {}


def _drive(d):
    """(P_l, P_r, [(left, right)] * NMAX) of drive d."""
    if d not in _FRAMES:
        w, h, seed, r, t, cal = DRIVES[d]
        base = synth.stereo_unit(w, h, seed, cal=cal)
        fr = [(base["l0"], base["r0"])]
        for k in range(1, NMAX):
            u = synth.stereo_unit(w, h, seed, cal=cal, rvec=np.array(r) * k, tvec=np.array(t) * k)
            fr.append((u["l1"], u["r1"]))
        _FRAMES[d] = (base["P_l"], base["P_r"], fr)
    return _FRAMES[d]


def _context():
    from visual_odom_b200.capi import Context
    return Context(0, max_features=8192)


def _alone(ctx, d, mono=False):
    """vo_seq_begin / vo_seq_push of drive d (NMAX frames): per frame (record, state, pose)."""
    P_l, P_r, fr = _drive(d)
    ctx.set_option("mono_rotation", 1 if mono else 0)
    try:
        ctx.seq_begin(fr[0][0], fr[0][1], P_l, P_r)
        return [(ctx.seq_push(*fr[k], mono=mono), ctx.seq_state(), ctx.seq_pose()) for k in range(1, NMAX)]
    finally:
        ctx.set_option("mono_rotation", 0)


@pytest.fixture(scope="module")
def alone(built):
    """Each drive alone on a fresh context, with and without the mono branch (computed on first use)."""
    cache = {}

    def get(d, mono=False):
        if (d, mono) not in cache:
            c = _context()
            cache[(d, mono)] = _alone(c, d, mono)
            c.close()
        return cache[(d, mono)]
    return get


def _run(ctx, n_slots, sched, pipelined=False, mono=False, bgr=False, env=ENV, submit=None):
    """Opens n_slots slots and runs the schedule: (slot, k0, drive, length) starts `drive` in `slot` at submission k0
    (its frame 0), frame j goes at submission k0 + j, and a slot with no frame gets a NULL pair.  Per submission:
    (records, [state of q], [pose of q]); state / pose only for submit-then-wait runs.  submit(k, lefts, rights, start)
    replaces ctx.mseq_submit."""
    img = (lambda a: np.repeat(a[:, :, None], 3, axis=2)) if bgr else (lambda a: a)
    ctx.mseq_open(n_slots, *env, mono_rotation=mono)
    K = max(k0 + L - 1 for _, k0, _, L in sched)

    def pairs(k):
        lefts, rights, start = [None] * n_slots, [None] * n_slots, {}
        for q, k0, d, L in sched:
            if k0 <= k < k0 + L:
                P_l, P_r, fr = _drive(d)
                lefts[q], rights[q] = img(fr[k - k0][0]), img(fr[k - k0][1])
                if k == k0:
                    start[q] = (P_l, P_r)
        return lefts, rights, start

    def go(k):
        lefts, rights, start = pairs(k)
        (submit or (lambda k, l, r, s: ctx.mseq_submit(l, r, start=s)))(k, lefts, rights, start)

    out = []
    if pipelined:
        go(1)
        for k in range(1, K + 1):
            if k + 1 <= K:
                go(k + 1)
            out.append((ctx.mseq_wait(mono=mono), None, None))
        return out
    for k in range(1, K + 1):
        go(k)
        recs = ctx.mseq_wait(mono=mono)
        out.append((recs, [ctx.mseq_state(q) for q in range(n_slots)], [ctx.mseq_pose(q) for q in range(n_slots)]))
    return out


def _same(a, b, where, keys=ARRAYS):
    for k in INTS:
        assert a[k] == b[k], f"{where}: {k} {a[k]} != {b[k]}"
    for k in keys:
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), f"{where}: {k}"


def _check(run, sched, alone, mono=False):
    """Every scheduled sequence against its drive alone; every slot without a sequence reports VO_MSEQ_RETIRED."""
    from visual_odom_b200 import capi
    n_slots = len(run[0][0])
    busy = set()
    for q, k0, d, L in sched:
        ref = alone(d, mono)
        recs, states, poses = run[k0 - 1]
        assert recs[q]["status"] == capi.VO_MSEQ_STARTED, f"drive {d} in slot {q} at {k0}"
        assert all(recs[q][k] == 0 for k in INTS) and not recs[q]["R"].any() and len(recs[q]["l0"]) == 0
        if mono:
            assert recs[q]["mono"]["status"] == 0 and not recs[q]["mono"]["R"].any() and len(recs[q]["ess_mask"]) == 0
        if states is not None:
            pts, ages, t = states[q]
            assert len(pts) == 0 and len(ages) == 0 and not t.any(), f"drive {d}: state after its start"
            assert np.array_equal(poses[q], np.eye(4)), f"drive {d}: pose after its start"
        busy.add((q, k0))
        for j in range(1, L):
            busy.add((q, k0 + j))
            recs, states, poses = run[k0 + j - 1]
            rec, st, pose = ref[j - 1]
            where = f"drive {d} in slot {q}, frame {j} (submission {k0 + j})"
            assert recs[q]["status"] == capi.VO_OK, where
            _same(recs[q], rec, where)
            if mono:
                for key in ("status", "n_inliers", "ransac_iters", "n_good"):
                    assert recs[q]["mono"][key] == rec["mono"][key], f"{where}: mono {key}"
                for key in ("R", "t"):
                    assert np.array_equal(recs[q]["mono"][key], rec["mono"][key]), f"{where}: mono {key}"
                assert np.array_equal(recs[q]["ess_mask"], rec["ess_mask"]), f"{where}: essential mask"
            if states is not None:
                for name, a, b in zip(("points", "ages", "translation"), states[q], st):
                    assert a.dtype == b.dtype and np.array_equal(a, b), f"{where}: carried {name}"
                assert np.array_equal(poses[q], pose), f"{where}: frame_pose"
        assert ref[-1][0]["n_valid"] > 30 and ref[-1][0]["n_inliers"] > 10
    for k, (recs, _, _) in enumerate(run, start=1):
        for q in range(n_slots):
            if (q, k) not in busy:
                assert recs[q]["status"] == capi.VO_MSEQ_RETIRED, f"empty slot {q} at submission {k}"


def _same_runs(a, b, what):
    for k, ((ra, sa, pa), (rb, sb, pb)) in enumerate(zip(a, b), start=1):
        for q in range(len(ra)):
            assert ra[q]["status"] == rb[q]["status"], f"{what}: slot {q} submission {k}"
            _same(ra[q], rb[q], f"{what}: slot {q} submission {k}")
            if sa is not None and sb is not None:
                assert np.array_equal(pa[q], pb[q]) and all(np.array_equal(x, y) for x, y in zip(sa[q], sb[q]))


# (slot, k0, drive, length)
EMPTY = [(0, 1, 0, 5), (2, 2, 1, 5), (1, 4, 2, 4)]
LATE = [(0, 1, 0, 3), (1, 1, 1, 6), (0, 6, 6, 4)]                  # slot 0 retired at 4, started at 6
FLIGHT = [(0, 1, 0, 3), (1, 1, 1, 6), (0, 5, 6, 4)]                # slot 0 retired at 4 (in flight), started at 5
REPLACE = [(0, 1, 0, 4), (1, 1, 1, 6), (0, 5, 7, 4)]               # drive 7 follows drive 0 directly, another calibration
LARGER = [(0, 1, 2, 4), (1, 1, 1, 6), (0, 5, 3, 5), (2, 2, 4, 5)]  # 512 x 200 after 656 x 248; 656 x 200 raises the grid


def test_starts_into_empty_slots_of_an_opened_run(ctx, alone):
    _check(_run(ctx, 3, EMPTY), EMPTY, alone)


@pytest.mark.parametrize("sched", [LATE, FLIGHT, REPLACE], ids=["retired-before", "retired-in-flight", "replaces-live"])
def test_a_start_into_a_used_slot_submit_then_wait_and_pipelined(ctx, alone, sched):
    """A retired slot restarted later, the slot retired by the submission in flight, and a live sequence replaced by one
    with another calibration: with two submissions in flight the old sequence's last frames (which still read the slot's
    calibration and carried translation) and the new one's first frames match their solo runs."""
    plain = _run(ctx, 2, sched)
    _check(plain, sched, alone)
    piped = _run(ctx, 2, sched, pipelined=True)
    _check(piped, sched, alone)
    _same_runs(piped, plain, "pipelined")


def test_a_smaller_image_after_a_larger_one_and_a_larger_bucket_grid(ctx, alone):
    for graphs in (1, 0):
        ctx.set_option("graphs", graphs)
        try:
            _check(_run(ctx, 3, LARGER), LARGER, alone)
            _check(_run(ctx, 3, LARGER, pipelined=True), LARGER, alone)
        finally:
            ctx.set_option("graphs", 1)
    assert max(r[0]["n_features"] for r in alone(4)) > 308


def test_mono_rotation_runs(ctx, alone):
    from visual_odom_b200 import capi
    sched = [(0, 1, 0, 4), (1, 2, 1, 5), (0, 5, 7, 4)]
    _check(_run(ctx, 3, sched, mono=True), sched, alone, mono=True)

    def submit(k, lefts, rights, start):
        if k == 3:            # the mono scratch holds the envelope's bucket grid: 656 x 200 needs more
            P_l, P_r, fr = _drive(4)
            with pytest.raises(capi.VoError) as e:
                ctx.mseq_submit(lefts[:2] + [fr[0][0]], rights[:2] + [fr[0][1]], start={2: (P_l, P_r)})
            assert e.value.code == capi.VO_E_CAPACITY and "mono scratch" in str(e.value)
        ctx.mseq_submit(lefts, rights, start=start)

    _check(_run(ctx, 3, sched, mono=True, pipelined=True, submit=submit), sched, alone, mono=True)


def test_colour_input_and_graphs_off_give_the_same_bits(ctx, alone):
    ref = _run(ctx, 3, FLIGHT + [(2, 2, 5, 4)])
    _check(ref, FLIGHT + [(2, 2, 5, 4)], alone)
    _same_runs(_run(ctx, 3, FLIGHT + [(2, 2, 5, 4)], bgr=True), ref, "BGR")
    ctx.set_option("graphs", 0)
    try:
        _same_runs(_run(ctx, 3, FLIGHT + [(2, 2, 5, 4)]), ref, "graphs 0")
    finally:
        ctx.set_option("graphs", 1)


def _queue(lengths, n_slots, drives):
    """Each drive starts in the first slot that frees (lowest index first), in order: the schedule."""
    free_at = [1] * n_slots
    sched = []
    for i, L in enumerate(lengths):
        q = min(range(n_slots), key=lambda s: (free_at[s], s))
        sched.append((q, free_at[q], drives[i % len(drives)], L))
        free_at[q] += L
    return sched


def test_several_starts_in_one_submission_and_a_queue_through_three_slots(ctx, alone):
    lengths = [6, 3, 5, 2, 4, 6, 3, 5, 4, 2]
    sched = _queue(lengths, 3, list(range(len(DRIVES))))
    assert sum(1 for s in sched if s[1] == 1) == 3                    # three starts in the first submission
    assert len({s[1] for s in sched}) < len(sched)                    # and again later
    _check(_run(ctx, 3, sched), sched, alone)
    _check(_run(ctx, 3, sched, pipelined=True), sched, alone)


def test_launch_counts(ctx):
    """Plain submissions of an opened run cost the launches of one vo_seq_submit and of a vo_mseq_begin run; a
    submission with starts at most one more."""
    d = [0, 1, 6]
    counts = {}

    def submit(k, lefts, rights, start):
        l0 = ctx.kernel_launches()
        ctx.mseq_submit(lefts, rights, start=start)
        counts.setdefault(k, ctx.kernel_launches() - l0)

    sched = [(0, 1, 0, 6), (1, 1, 1, 3), (2, 2, 6, 5), (1, 4, 6, 3)]
    _run(ctx, 3, sched, submit=submit)
    ref_plain = counts[5]
    assert counts[3] == counts[6] == ref_plain > 0
    assert all(counts[k] <= ref_plain + 1 for k in (1, 2, 4)), counts
    # vo_seq_* and a vo_mseq_begin run at the same steps
    P_l, P_r, fr = _drive(0)
    ctx.seq_begin(fr[0][0], fr[0][1], P_l, P_r)
    for k in (1, 2):
        ctx.seq_push(*fr[k])
    l0 = ctx.kernel_launches()
    ctx.seq_push(*fr[3])
    assert ctx.kernel_launches() - l0 == ref_plain
    frs = [_drive(x)[2] for x in d]
    ctx.mseq_begin([f[0][0] for f in frs], [f[0][1] for f in frs], np.stack([_drive(x)[0] for x in d]),
                   np.stack([_drive(x)[1] for x in d]))
    for k in (1, 2):
        ctx.mseq_submit([f[k][0] for f in frs], [f[k][1] for f in frs]); ctx.mseq_wait(want_points=False)
    l0 = ctx.kernel_launches()
    ctx.mseq_submit([f[3][0] for f in frs], [f[3][1] for f in frs]); ctx.mseq_wait(want_points=False)
    assert ctx.kernel_launches() - l0 == ref_plain


def test_a_started_sequence_matches_the_reference_path(ctx):
    """Drive 1 started at submission 3 in slot 1 of an opened run, frame by frame against cv2 through the reference's
    glue (oracle/ref_path.py)."""
    pytest.importorskip("cv2")
    from oracle import ref_path
    sched = [(0, 1, 0, 5), (1, 3, 1, 5)]
    run = _run(ctx, 2, sched)
    P_l, P_r, fr = _drive(1)
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    for j in range(1, 5):
        (l0, r0), (l1, r1) = fr[j - 1], fr[j]
        recs, states, poses = run[3 + j - 1]
        got = recs[1]
        pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend="cv2")
        X = ref_path.triangulate(P_l, P_r, pL0, pR0, "cv2")
        R, translation, inl, rvec = ref_path.tracking_frame2frame(P_l, pL0, pL1, X, translation, "cv2")
        assert got["n_features"] == len(info["bucketed"]) and got["n_tracked"] == len(info["kept_idx"])
        assert got["n_valid"] == len(pL0)
        for name, ref in (("l0", pL0), ("r0", pR0), ("l1", pL1), ("r1", pR1)):
            assert np.array_equal(got[name], ref), f"frame {j}: {name}"
        assert got["n_inliers"] == len(inl), f"frame {j}: inlier count"
        assert np.linalg.norm(got["R"] - R) / np.linalg.norm(R) <= 1e-4
        assert np.linalg.norm(got["tvec"] - translation) / np.linalg.norm(translation) <= 1e-4
        frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
        assert np.abs(poses[1] - frame_pose).max() <= 1e-6 * max(1.0, np.abs(frame_pose).max()), f"frame {j}: frame_pose"
        pts, ages, _ = states[1]
        assert np.array_equal(pts, fs.points) and np.array_equal(ages, fs.ages), f"frame {j}: carried FeatureSet"


def _starts(*items):
    from visual_odom_b200.capi import VoMseqStart
    arr = (VoMseqStart * max(len(items), 1))()
    for s, (q, w, h, d) in zip(arr, items):
        P_l, P_r, _ = _drive(d)
        s.slot, s.w, s.h = q, w, h
        s.P_l[:] = np.asarray(P_l, np.float32).reshape(12).tolist()
        s.P_r[:] = np.asarray(P_r, np.float32).reshape(12).tolist()
    return arr, len(items)


def test_refusals_change_nothing(ctx, alone):
    """Every refusal of vo_mseq_submit_start and vo_mseq_open, in the middle of a pipelined run with a submission in flight;
    the run then goes on bit for bit."""
    from visual_odom_b200 import capi
    lib, h = ctx.lib, ctx.h
    I, U = capi.VO_E_INVALID, capi.VO_E_UNSUPPORTED
    sched = [(0, 1, 0, 5), (1, 2, 1, 4)]
    big = np.zeros((260, 700), np.uint8)

    def refuse(k, lefts, rights, start):
        if k == 3:            # submission 2 is in flight; slot 2 is empty, slot 1 live
            fr = _drive(2)[2][0]
            keep = [a for a in lefts if a is not None] + [fr[0], fr[1], big]
            lp = (C.c_void_p * 3)(*[None if a is None else a.ctypes.data for a in lefts])
            rp = (C.c_void_p * 3)(*[None if a is None else a.ctypes.data for a in rights])
            pa = np.array([a.shape[1] if a is not None else 0 for a in lefts], np.uint64)

            def try_start(st, ch=1, pitch=None, l2=fr[0], r2=fr[1], w2=656):
                lp[2] = None if l2 is None else l2.ctypes.data
                rp[2] = None if r2 is None else r2.ctypes.data
                p = pa.copy(); p[2] = w2 if pitch is None else pitch
                arr, n = st
                return lib.vo_mseq_submit_start(h, lp, rp, p.ctypes.data, ch, n, arr)

            assert try_start(_starts((3, 656, 248, 2))) == I                       # slot out of range
            assert try_start(_starts((-1, 656, 248, 2))) == I
            assert try_start(_starts((2, 656, 248, 2), (2, 656, 248, 2))) == I     # two starts in one slot
            assert try_start(_starts((2, 656, 248, 2)), l2=None) == I              # one image
            assert try_start(_starts((2, 656, 248, 2)), l2=None, r2=None) == I     # no pair
            assert try_start(_starts((2, 656, 248, 2)), pitch=655) == I            # pitch < w
            assert try_start(_starts((2, 656, 248, 2)), ch=3) == I                 # BGR needs 3 w
            assert try_start(_starts((2, 0, 248, 2))) == I and try_start(_starts((2, 656, -1, 2))) == I
            assert lib.vo_mseq_submit_start(h, lp, rp, pa.ctypes.data, 1, -1, None) == I
            assert try_start(_starts((2, 700, 248, 2)), l2=big, r2=big, w2=700) == U   # outside the envelope
            assert try_start(_starts((2, 656, 260, 2)), l2=big, r2=big, w2=700) == U
            assert try_start(_starts((2, 160, 200, 2))) == U                       # one pyramid level less
            assert "pyramid" in lib.vo_last_error(h).decode()
            assert try_start(_starts((2, 656, 9, 2))) == U                         # rows / 10 == 0
            # a plain submission still refuses a pair for an empty slot
            p = pa.copy(); p[2] = 656
            assert lib.vo_mseq_submit_sized(h, lp, rp, p.ctypes.data, 1) == I
            assert "retired" in lib.vo_last_error(h).decode()
            # (vo_mseq_open ends a running multi-sequence run, so only its argument refusals are tried here)
            assert lib.vo_mseq_open(h, 0, 656, 248, 0) == I
            assert lib.vo_mseq_open(h, capi.VO_MSEQ_MAX + 1, 656, 248, 0) == I
            assert lib.vo_mseq_open(h, 2, 0, 248, 0) == I and lib.vo_mseq_open(h, 2, 656, 248, 4) == I
            del keep
        ctx.mseq_submit(lefts, rights, start=start)

    run = _run(ctx, 3, sched, pipelined=True, submit=refuse)
    _check(run, sched, alone)
    # a third submission in flight
    ctx.mseq_open(2, *ENV)
    P_l, P_r, fr = _drive(0)
    ctx.mseq_submit([fr[0][0], None], [fr[0][1], None], start={0: (P_l, P_r)})
    ctx.mseq_submit([fr[1][0], None], [fr[1][1], None])
    arr, n = _starts((1, 640, 240, 0))
    lp = (C.c_void_p * 2)(fr[2][0].ctypes.data, fr[0][0].ctypes.data)
    rp = (C.c_void_p * 2)(fr[2][1].ctypes.data, fr[0][1].ctypes.data)
    assert lib.vo_mseq_submit_start(h, lp, rp, np.array([640, 640], np.uint64).ctypes.data, 1, n, arr) == I
    ctx.mseq_wait(); ctx.mseq_wait()


def test_a_run_begun_with_one_size_starts_only_that_size(ctx, alone):
    from visual_odom_b200 import capi
    P_l, P_r, fr = _drive(0)
    P1, P1r, fr1 = _drive(6)                              # 640 x 240 as drive 0
    ctx.mseq_begin([fr[0][0], fr[0][0]], [fr[0][1], fr[0][1]], P_l, P_r)
    ctx.mseq_submit([fr[1][0], None], [fr[1][1], None])
    ctx.mseq_wait()
    with pytest.raises(capi.VoError):
        ctx.mseq_submit([fr[2][0], _drive(1)[2][0][0]], [fr[2][1], _drive(1)[2][0][1]], start={1: _drive(1)[:2]})
    err = ctx.lib.vo_last_error(ctx.h).decode()
    assert "vo_mseq_open" in err and "vo_mseq_begin_sized" in err, err
    out = []
    for j in range(0, 5):
        ctx.mseq_submit([fr[2 + j][0] if 2 + j < NMAX else None, fr1[j][0]], [fr[2 + j][1] if 2 + j < NMAX else None, fr1[j][1]],
                        start={1: (P1, P1r)} if j == 0 else None)
        out.append(ctx.mseq_wait())
    assert out[0][1]["status"] == capi.VO_MSEQ_STARTED
    ref = alone(6)
    for j in range(1, 5):
        _same(out[j][1], ref[j - 1][0], f"frame {j}")
    ref0 = alone(0)
    for j in range(0, 4):
        _same(out[j][0], ref0[j + 1][0], f"drive 0 frame {j + 2}")
