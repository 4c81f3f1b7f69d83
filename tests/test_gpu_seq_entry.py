"""The entry points of the streaming sequence modes (vo_seq_*, vo_mseq_*): every refusal as one table -- each row one call
with one fault, its code and a message substring -- after which the context runs sequences as a fresh one does; and the
begin calls refused while a vo_batch_submit submission has not been waited for, which that submission survives bit for
bit."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from visual_odom_b200 import capi, synth

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H, NF = 320, 120, 5
STEP = ((0.001, -0.004, 0.0005), (0.01, -0.003, -0.2))
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
ARRAYS = ("rvec", "tvec", "R", "l0", "r0", "l1", "r1")


def _frames(seed):
    base = synth.stereo_unit(W, H, seed)
    out = [(base["l0"], base["r0"])]
    for k in range(1, NF):
        u = synth.stereo_unit(W, H, seed, rvec=np.array(STEP[0]) * k, tvec=np.array(STEP[1]) * k)
        out.append((u["l1"], u["r1"]))
    return base, out


@pytest.fixture(scope="module")
def drives():
    (base, a), (_, b) = _frames(3), _frames(7)
    return base["P_l"], base["P_r"], a, b


def _short_runs(c, P_l, P_r, a, b):
    """One sequence pushed frame by frame, then two in lockstep with two submissions in flight."""
    c.seq_begin(a[0][0], a[0][1], P_l, P_r)
    single = [c.seq_push(l, r) for l, r in a[1:]]
    c.mseq_begin([a[0][0], b[0][0]], [a[0][1], b[0][1]], P_l, P_r)
    multi = []
    c.mseq_submit([a[1][0], b[1][0]], [a[1][1], b[1][1]])
    for k in range(1, NF):
        if k + 1 < NF:
            c.mseq_submit([a[k + 1][0], b[k + 1][0]], [a[k + 1][1], b[k + 1][1]])
        multi += c.mseq_wait()
    return single + multi, [c.mseq_pose(q) for q in range(2)]


def _same_runs(got, want):
    for i, (x, y) in enumerate(zip(got[0], want[0])):
        for k in INTS:
            assert x[k] == y[k], (i, k)
        for k in ARRAYS:
            assert np.array_equal(x[k], y[k]), (i, k)
    assert len(got[0]) == len(want[0]) and all(np.array_equal(x, y) for x, y in zip(got[1], want[1]))


@pytest.fixture(scope="module")
def fresh_runs(built, drives):
    c = capi.Context(0, max_features=2048)
    runs = _short_runs(c, *drives)
    c.close()
    assert all(r["n_valid"] > 0 and r["n_inliers"] > 0 for r in runs[0])
    return runs


def _args(P_l, P_r, a, b):
    """The pointers and buffers the rows pass: host frames 0 .. 2 of sequence a (l*, r*), pair tables of two sequences
    (lp* / rp*), a table with one image of sequence 1 missing, sequence 1 retired, device images, result buffers."""
    def tab(*ptrs):
        return (C.c_void_p * len(ptrs))(*ptrs)
    t = SimpleNamespace()
    t.Pl = np.ascontiguousarray(P_l, np.float32).reshape(12); t.Pr = np.ascontiguousarray(P_r, np.float32).reshape(12)
    t.Pl2 = np.concatenate([t.Pl, t.Pl]); t.Pr2 = np.concatenate([t.Pr, t.Pr])
    t.imgs = [np.ascontiguousarray(x) for fr in (a, b) for pair in fr[:3] for x in pair]
    p = [x.ctypes.data for x in t.imgs]                 # a: frames 0, 1, 2 at 0..5 (left, right); b: at 6..11
    t.l0, t.r0, t.l1, t.r1 = p[0], p[1], p[2], p[3]
    t.lp0, t.rp0 = tab(p[0], p[6]), tab(p[1], p[7])
    t.lp1, t.rp1 = tab(p[2], p[8]), tab(p[3], p[9])
    t.lp2, t.rp2 = tab(p[4], p[10]), tab(p[5], p[11])
    t.rp0_half, t.rp1_half = tab(p[1], None), tab(p[3], None)
    t.dev = [torch.from_numpy(x).cuda() for x in t.imgs[2:4]]
    t.dl, t.dr = (capi.image_descriptor(d.shape, d.stride(), d.data_ptr())[0] for d in t.dev)
    t.res = (capi.VoUnitResult * 2)(); t.mono = (capi.VoMonoResult * 2)()
    t.st = np.zeros(2, np.int32); t.pose = np.zeros(16)
    return t


def _rows(t):
    """(state, entry point, arguments after the context, code, message substring).  States: "none" (nothing begun),
    "seq" / "mseq" (one / two sequences begun and idle), a digit (frames in flight), "mseq_retired" (sequence 1 retired),
    "mono_opt" (the option "mono_rotation" set)."""
    I, U, K = capi.VO_E_INVALID, capi.VO_E_UNSUPPORTED, capi.VO_E_CAPACITY
    Pl, Pr, res, st, mono = capi._p(t.Pl), capi._p(t.Pr), t.res, capi._p(t.st), t.mono
    dl, dr, pose = C.byref(t.dl), C.byref(t.dr), capi._p(t.pose)
    seq0 = (W, H, Pl, Pr, t.l0, t.r0, W)
    mseq0 = (2, W, H, Pl, Pr, t.lp0, t.rp0, W, 1)
    return [
        # not begun
        ("none", "vo_seq_submit", (t.l1, t.r1, W, 1), I, "call vo_seq_begin first"),
        ("none", "vo_seq_submit_device", (dl, dr), I, "call vo_seq_begin first"),
        ("none", "vo_seq_wait", (res, None, 0), I, "no frame in flight"),
        ("none", "vo_seq_wait_mono", (res, mono, None, 0, None, 0), I, "no frame in flight"),
        ("none", "vo_mseq_submit", (t.lp1, t.rp1, W, 1), I, "call vo_mseq_begin first"),
        ("none", "vo_mseq_wait", (res, st, None, 0), I, "call vo_mseq_begin first"),
        ("none", "vo_mseq_wait_mono", (res, st, mono, None, 0, None, 0), I, "call vo_mseq_begin first"),
        ("none", "vo_mseq_state", (0, None, None, 0, None, None, None), I, "call vo_mseq_begin first"),
        ("none", "vo_mseq_pose", (0, pose), I, "call vo_mseq_begin first"),
        # the other mode's frame calls, and its begin while frames are in flight
        ("mseq", "vo_seq_submit", (t.l1, t.r1, W, 1), I, "begun with vo_mseq_begin"),
        ("mseq", "vo_seq_submit_device", (dl, dr), I, "begun with vo_mseq_begin"),
        ("mseq", "vo_seq_push", (t.l1, t.r1, W, res, None, 0), I, "begun with vo_mseq_begin"),
        ("mseq", "vo_seq_wait", (res, None, 0), I, "begun with vo_mseq_begin"),
        ("mseq", "vo_seq_wait_mono", (res, mono, None, 0, None, 0), I, "begun with vo_mseq_begin"),
        ("mseq", "vo_seq_state", (None, None, 0, None, None, None), I, "begun with vo_mseq_begin"),
        ("seq", "vo_mseq_submit", (t.lp1, t.rp1, W, 1), I, "begun with vo_seq_begin"),
        ("seq", "vo_mseq_wait", (res, st, None, 0), I, "begun with vo_seq_begin"),
        ("seq", "vo_mseq_wait_mono", (res, st, mono, None, 0, None, 0), I, "begun with vo_seq_begin"),
        ("seq", "vo_mseq_state", (0, None, None, 0, None, None, None), I, "begun with vo_seq_begin"),
        ("seq", "vo_mseq_pose", (0, pose), I, "begun with vo_seq_begin"),
        ("mseq1", "vo_seq_begin", seq0, I, "have not been waited for"),
        ("seq1", "vo_mseq_begin", mseq0, I, "have not been waited for"),
        # a third submission, a push over a frame in flight, a wait with nothing in flight
        ("seq2", "vo_seq_submit", (t.l1, t.r1, W, 1), I, "in flight"),
        ("seq2", "vo_seq_submit_device", (dl, dr), I, "in flight"),
        ("mseq2", "vo_mseq_submit", (t.lp1, t.rp1, W, 1), I, "in flight"),
        ("seq1", "vo_seq_push", (t.l1, t.r1, W, res, None, 0), I, "in flight"),
        ("seq", "vo_seq_wait", (res, None, 0), I, "no frame in flight"),
        ("seq", "vo_seq_wait_mono", (res, mono, None, 0, None, 0), I, "no frame in flight"),
        ("mseq", "vo_mseq_wait", (res, st, None, 0), I, "in flight"),
        ("mseq", "vo_mseq_wait_mono", (res, st, mono, None, 0, None, 0), I, "in flight"),
        # NULL results
        ("seq1", "vo_seq_wait", (None, None, 0), I, "null result"),
        ("seq1", "vo_seq_wait_mono", (res, None, None, 0, None, 0), I, "null result"),
        ("seq", "vo_seq_push", (t.l1, t.r1, W, None, None, 0), I, "null result"),
        ("mseq1", "vo_mseq_wait", (None, st, None, 0), I, "null result"),
        ("mseq1", "vo_mseq_wait", (res, None, None, 0), I, "null result"),
        ("mseq1", "vo_mseq_wait_mono", (res, st, None, None, 0, None, 0), I, "null result"),
        # channels = 2
        ("seq", "vo_seq_begin_ex", (W, H, Pl, Pr, t.l0, t.r0, 2 * W, 2), I, "channels"),
        ("seq", "vo_seq_submit", (t.l1, t.r1, 2 * W, 2), I, "channels"),
        ("seq", "vo_seq_push_ex", (t.l1, t.r1, 2 * W, 2, res, None, 0), I, "channels"),
        ("none", "vo_mseq_begin", (2, W, H, Pl, Pr, t.lp0, t.rp0, 2 * W, 2), I, "channels"),
        ("mseq", "vo_mseq_submit", (t.lp1, t.rp1, 2 * W, 2), I, "channels"),
        # a pitch below w * channels, NULL images
        ("seq", "vo_seq_begin", (W, H, Pl, Pr, t.l0, t.r0, W - 1), I, "bad argument"),
        ("seq", "vo_seq_begin_ex", (W, H, Pl, Pr, t.l0, t.r0, 3 * W - 1, 3), I, "bad argument"),
        ("seq", "vo_seq_begin", (W, H, Pl, Pr, None, t.r0, W), I, "bad argument"),
        ("seq", "vo_seq_submit", (t.l1, t.r1, W - 1, 1), I, "bad argument"),
        ("seq", "vo_seq_submit", (t.l1, None, W, 1), I, "bad argument"),
        ("mseq", "vo_mseq_begin", (2, W, H, Pl, Pr, t.lp0, t.rp0, W - 1, 1), I, "bad argument"),
        ("mseq", "vo_mseq_begin", (2, W, H, Pl, Pr, None, t.rp0, W, 1), I, "bad argument"),
        ("mseq", "vo_mseq_submit", (t.lp1, t.rp1, W - 1, 1), I, "bad argument"),
        # h < 10: no rows/10 bucket
        ("seq", "vo_seq_begin", (W, 9, Pl, Pr, t.l0, t.r0, W), U, "rows/10"),
        ("seq", "vo_seq_begin_device", (W, 9, Pl, Pr, dl, dr), U, "rows/10"),
        ("mseq", "vo_mseq_begin", (2, W, 9, Pl, Pr, t.lp0, t.rp0, W, 1), U, "rows/10"),
        # NULL matrices
        ("seq", "vo_seq_begin", (W, H, None, Pr, t.l0, t.r0, W), I, "bad argument"),
        ("seq", "vo_seq_begin_ex", (W, H, Pl, None, t.l0, t.r0, W, 1), I, "bad argument"),
        ("seq", "vo_seq_begin_device", (W, H, None, Pr, dl, dr), I, "bad argument"),
        ("mseq", "vo_mseq_begin", (2, W, H, None, Pr, t.lp0, t.rp0, W, 1), I, "bad argument"),
        ("mseq", "vo_mseq_begin_ex", (2, W, H, Pl, None, t.lp0, t.rp0, W, 1, 0), I, "bad argument"),
        ("mseq", "vo_mseq_begin_calib", (2, W, H, capi._p(t.Pl2), None, t.lp0, t.rp0, W, 1, 0), I, "bad argument"),
        # sequence counts, flags, the context option
        ("none", "vo_mseq_begin", (0, W, H, Pl, Pr, t.lp0, t.rp0, W, 1), I, "n_seq = 0"),
        ("none", "vo_mseq_begin", (capi.VO_MSEQ_MAX + 1, W, H, Pl, Pr, t.lp0, t.rp0, W, 1), K, f"n_seq = {capi.VO_MSEQ_MAX + 1}"),
        ("none", "vo_mseq_begin_ex", (2, W, H, Pl, Pr, t.lp0, t.rp0, W, 1, 2), I, "unknown flag bits 0x2"),
        ("mono_opt", "vo_mseq_begin", mseq0, U, "mono_rotation"),
        # a pair with one image, a retired sequence
        ("none", "vo_mseq_begin", (2, W, H, Pl, Pr, t.lp0, t.rp0_half, W, 1), I, "sequence 1 has no first pair"),
        ("mseq", "vo_mseq_submit", (t.lp1, t.rp1_half, W, 1), I, "sequence 1 has only one image"),
        ("mseq_retired", "vo_mseq_submit", (t.lp2, t.rp2, W, 1), I, "sequence 1 was retired"),
        # a bad q
        ("mseq", "vo_mseq_state", (2, None, None, 0, None, None, None), I, "bad sequence index 2"),
        ("mseq", "vo_mseq_state", (-1, None, None, 0, None, None, None), I, "bad sequence index -1"),
        ("mseq", "vo_mseq_pose", (2, pose), I, "bad argument"),
        ("mseq", "vo_mseq_pose", (0, None), I, "bad argument"),
        # the mono result of sequences begun without the branch
        ("seq1", "vo_seq_wait_mono", (res, mono, None, 0, None, 0), I, "mono_rotation"),
        ("mseq1", "vo_mseq_wait_mono", (res, st, mono, None, 0, None, 0), I, "VO_MSEQ_MONO_ROTATION"),
    ]


def _enter(c, state, P_l, P_r, a, b):
    """Puts c into `state`; returns the number of frames left in flight."""
    kind, inflight = (state[:-1], int(state[-1])) if state[-1].isdigit() else (state, 0)
    if kind == "seq":
        c.seq_begin(a[0][0], a[0][1], P_l, P_r)
        for k in range(1, 1 + inflight):
            c.seq_submit(*a[k])
    elif kind in ("mseq", "mseq_retired"):
        c.mseq_begin([a[0][0], b[0][0]], [a[0][1], b[0][1]], P_l, P_r)
        for k in range(1, 1 + inflight):
            c.mseq_submit([a[k][0], b[k][0]], [a[k][1], b[k][1]])
        if kind == "mseq_retired":
            c.mseq_submit([a[1][0], None], [a[1][1], None])
            assert c.mseq_wait()[1]["status"] == capi.VO_MSEQ_RETIRED
    elif kind == "mono_opt":
        c.set_option("mono_rotation", 1)
    return inflight


def test_refusal_table(built, drives, fresh_runs):
    P_l, P_r, a, b = drives
    c, idle = capi.Context(0, max_features=2048), capi.Context(0, max_features=2048)      # idle: nothing is ever begun
    t = _args(P_l, P_r, a, b)
    for state, name, args, code, msg in _rows(t):
        ctx = idle if state == "none" else c
        inflight = _enter(ctx, state, P_l, P_r, a, b)
        rc = getattr(ctx.lib, name)(ctx.h, *args)
        err = ctx.lib.vo_last_error(ctx.h).decode()
        assert rc == code and msg in err, f"{name} in state {state}: {rc}, {err!r}; expected {code}, {msg!r}"
        if state == "mono_opt":
            ctx.set_option("mono_rotation", 0)
        for _ in range(inflight):           # the refused call left the frames in flight as they were
            ctx.mseq_wait() if state.startswith("mseq") else ctx.seq_wait()
    _same_runs(_short_runs(c, P_l, P_r, a, b), fresh_runs)
    c.close(); idle.close()


def test_begin_is_refused_while_a_batch_submission_is_pending(built, drives, fresh_runs):
    """Every begin call would upload into the unit buffers, rebuild their pyramids and may re-allocate the pinned block
    that receives the submission's records; it is refused before it changes anything."""
    P_l, P_r, a, b = drives
    units = [dict(l0=a[0][0], r0=a[0][1], l1=a[1][0], r1=a[1][1], n_select=300, t_prev=(0.0, 0.0, -0.2)),
             dict(l0=b[1][0], r0=b[1][1], l1=b[2][0], r1=b[2][1], n_select=300, t_prev=(0.0, 0.0, -0.2))]

    def submit(c):
        c.batch_configure(W, H, 2, P_l, P_r)
        arr, keep, pitch = c.make_units(units)
        c.batch_submit(arr, 0, pitch)
        return arr, keep

    c, fresh = capi.Context(0, max_features=2048), capi.Context(0, max_features=2048)
    alive = submit(c)
    for begin in (lambda: c.seq_begin(a[0][0], a[0][1], P_l, P_r),
                  lambda: c.mseq_begin([a[0][0], b[0][0]], [a[0][1], b[0][1]], P_l, P_r)):
        with pytest.raises(capi.VoError, match="has not been waited for") as e:
            begin()
        assert e.value.code == capi.VO_E_INVALID
    got = c.batch_wait(0, 2, raw=True)
    alive_fresh = submit(fresh)
    want = fresh.batch_wait(0, 2, raw=True)
    for f in capi.RESULT_DTYPE.names:
        assert np.array_equal(got[f], want[f]), f
    assert (want["n_valid"] > 0).all() and (want["n_inliers"] > 0).all()
    del alive, alive_fresh
    _same_runs(_short_runs(c, P_l, P_r, a, b), fresh_runs)
    c.close(); fresh.close()
