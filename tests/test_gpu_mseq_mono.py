"""trackingFrame2Frame(mono_rotation = true) for every sequence of the multi-sequence mode (vo_mseq_begin_ex with the flag
VO_MSEQ_MONO_ROTATION, vo_mseq_wait_mono): each sequence's records, mono results, essential masks, point lists, carried
state and frame_pose are bit for bit those of running it alone through vo_seq_* with the option "mono_rotation" (which
tests/test_gpu_seq_mono.py pins to cv2), the PnP side is that of the same run without the flag, and pipelining, colour
input, graphs, a textureless and a retired sequence, the launch count, the refusals and re-begins on one context are
covered."""
import ctypes as C

import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

# (seed, per-frame rotation, per-frame translation)
DRIVES = [
    (31, (0.001, -0.004, 0.0005), (0.01, -0.003, -0.2)),
    (7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25)),
    (13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15)),
    (42, (0.003, -0.001, 0.0005), (0.015, 0.0, -0.3)),
    (5, (-0.001, -0.002, 0.001), (0.0, -0.005, -0.18)),
]
SETS = {"640x240": (640, 240, 10, 5), "1241x376": (1241, 376, 7, 3)}     # w, h, frames, drives
PNP_INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
PNP_ARRAYS = ("rvec", "tvec", "l0", "r0", "l1", "r1")
MONO_INTS = ("status", "n_inliers", "ransac_iters", "n_good")
MAX_FEATURES = 8192                     # that of the session's context


def _drive(seed, r, t, n, w, h):
    base = synth.stereo_unit(w, h, seed)
    out = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=np.array(r) * k, tvec=np.array(t) * k)
        out.append((u["l1"], u["r1"]))
    return base, out


@pytest.fixture(scope="module")
def sets():
    out = {}
    for name, (w, h, nf, nd) in SETS.items():
        d = [_drive(*x, n=nf, w=w, h=h) for x in DRIVES[:nd]]
        out[name] = (d[0][0]["P_l"], d[0][0]["P_r"], [fr for _, fr in d])
    return out


def _same(a, b, where, mono=True):
    """Records (R included) and, with mono, the mono results and essential masks, bit for bit."""
    for k in PNP_INTS:
        assert a[k] == b[k], f"{where}: {k} {a[k]} != {b[k]}"
    for k in PNP_ARRAYS + ("R",):
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), f"{where}: {k}"
    if mono:
        ma, mb = a["mono"], b["mono"]
        for k in MONO_INTS:
            assert ma[k] == mb[k], f"{where}: mono {k} {ma[k]} != {mb[k]}"
        assert np.array_equal(ma["R"], mb["R"]) and np.array_equal(ma["t"], mb["t"]), f"{where}: mono R / t"
        assert np.array_equal(a["ess_mask"], b["ess_mask"]), f"{where}: essential mask"


def _same_state(a, b, where):
    for name, x, y in zip(("points", "ages", "translation"), a, b):
        assert x.dtype == y.dtype and np.array_equal(x, y), f"{where}: carried {name}"


def _gray_or_bgr(im, bgr):
    return None if im is None else (np.repeat(im[:, :, None], 3, 2) if bgr else im)


def _run_mseq(c, P_l, P_r, frames, mono=True, pipelined=False, bgr=False, edit=None):
    """frames[q][k] = (left, right); edit(q, k, pair) -> pair changes or retires (None, None) a frame.  Per frame:
    (records, [state of q], [pose of q]); state / pose only for submit-then-wait runs, whose last entry is then also
    what a pipelined run ends with."""
    n, nf = len(frames), len(frames[0])
    pair = (lambda q, k: frames[q][k]) if edit is None else (lambda q, k: edit(q, k, frames[q][k]))
    c.mseq_begin([_gray_or_bgr(f[0][0], bgr) for f in frames], [_gray_or_bgr(f[0][1], bgr) for f in frames], P_l, P_r,
                 mono_rotation=mono)

    def submit(k):
        ps = [pair(q, k) for q in range(n)]
        c.mseq_submit([_gray_or_bgr(p[0], bgr) for p in ps], [_gray_or_bgr(p[1], bgr) for p in ps])

    out = []
    if pipelined:
        submit(1)
        for k in range(1, nf):
            if k + 1 < nf:
                submit(k + 1)
            out.append((c.mseq_wait(mono=mono), None, None))
        return out
    for k in range(1, nf):
        submit(k)
        recs = c.mseq_wait(mono=mono)
        out.append((recs, [c.mseq_state(q) for q in range(n)], [c.mseq_pose(q) for q in range(n)]))
    return out


def _run_alone(c, P_l, P_r, fr):
    """One sequence through vo_seq_* with the option "mono_rotation": per frame (record, state, pose)."""
    c.set_option("mono_rotation", 1)
    try:
        c.seq_begin(fr[0][0], fr[0][1], P_l, P_r)
        return [(c.seq_push(l, r, mono=True), c.seq_state(), c.seq_pose()) for l, r in fr[1:]]
    finally:
        c.set_option("mono_rotation", 0)


@pytest.fixture(scope="module")
def mono_runs(ctx, sets):
    return {name: _run_mseq(ctx, *s) for name, s in sets.items()}


def _check_run(got, want, n, where=""):
    """Two submit-then-wait mono runs: records, mono results, masks, states and poses bit for bit."""
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(got, want), start=1):
        for q in range(n):
            _same(a[q], b[q], f"{where}sequence {q} frame {k}")
            _same_state(sa[q], sb[q], f"{where}sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q]), f"{where}sequence {q} frame {k}: frame_pose"


@pytest.mark.parametrize("name", list(SETS))
def test_each_sequence_is_bit_identical_to_running_it_alone(ctx, sets, mono_runs, name):
    from visual_odom_b200 import capi
    P_l, P_r, frames = sets[name]
    got = mono_runs[name]
    for q, fr in enumerate(frames):
        alone = _run_alone(ctx, P_l, P_r, fr)
        for k, ((recs, states, poses), (a, st, pose)) in enumerate(zip(got, alone), start=1):
            r = recs[q]
            assert r["status"] == capi.VO_OK
            _same(r, a, f"sequence {q} frame {k}")
            _same_state(states[q], st, f"sequence {q} frame {k}")
            assert np.array_equal(poses[q], pose), f"sequence {q} frame {k}: frame_pose"
            assert r["mono"]["status"] == capi.VO_OK and np.array_equal(r["R"], r["mono"]["R"]), f"sequence {q} frame {k}"
            assert r["mono"]["n_inliers"] == int(r["ess_mask"].sum())
        assert a["n_valid"] > 50 and a["mono"]["n_inliers"] > 20
        assert np.linalg.norm(pose[:3, 3]) > 0.1                           # frame_pose was integrated
    # the sequences' RANSACs stop at different adaptive bounds within one launch
    iters = [[recs[q]["mono"]["ransac_iters"] for q in range(len(frames))] for recs, _, _ in got]
    assert any(len(set(row)) > 1 for row in iters), iters
    print(f"{name}: essential-matrix RANSAC iterations per frame and sequence {iters}")


@pytest.mark.parametrize("name", list(SETS))
def test_the_pnp_side_is_that_of_the_run_without_the_flag(ctx, sets, mono_runs, name):
    P_l, P_r, frames = sets[name]
    off = _run_mseq(ctx, P_l, P_r, frames, mono=False)
    for k, ((a, sa, _), (b, sb, _)) in enumerate(zip(mono_runs[name], off), start=1):
        for q in range(len(frames)):
            for key in PNP_INTS:
                assert a[q][key] == b[q][key], f"sequence {q} frame {k}: {key}"
            for key in PNP_ARRAYS:
                assert np.array_equal(a[q][key], b[q][key]), f"sequence {q} frame {k}: {key}"
            assert "mono" not in b[q]
            _same_state(sa[q], sb[q], f"sequence {q} frame {k}")


def test_pipelining_colour_and_graphs_change_nothing(built, ctx, sets, mono_runs):
    from visual_odom_b200.capi import Context
    P_l, P_r, frames = sets["640x240"]
    want = mono_runs["640x240"]
    n = len(frames)
    piped = _run_mseq(ctx, P_l, P_r, frames, pipelined=True)
    for k, ((a, _, _), (b, _, _)) in enumerate(zip(piped, want), start=1):
        for q in range(n):
            _same(a[q], b[q], f"pipelined: sequence {q} frame {k}")
    for q in range(n):
        assert np.array_equal(ctx.mseq_pose(q), want[-1][2][q])
        _same_state(ctx.mseq_state(q), want[-1][1][q], f"pipelined: sequence {q} at the end")
    _check_run(_run_mseq(ctx, P_l, P_r, frames, bgr=True), want, n, "BGR: ")
    c = Context(0, max_features=MAX_FEATURES)
    c.set_option("graphs", 0)
    try:
        _check_run(_run_mseq(c, P_l, P_r, frames), want, n, "graphs = 0: ")
    finally:
        c.close()


def test_a_textureless_or_retired_sequence_leaves_the_others_alone(ctx, sets, mono_runs):
    from visual_odom_b200 import capi
    P_l, P_r, frames = sets["640x240"]
    want = mono_runs["640x240"]
    h, w = frames[0][0][0].shape
    flat, gone, k_flat, k_gone = 1, 3, 4, 6
    blank = np.full((h, w), 128, np.uint8)

    def edit(q, k, pair):
        if q == flat and k in (k_flat, k_flat + 1):
            return blank, blank
        if q == gone and k >= k_gone:
            return None, None
        return pair

    got = _run_mseq(ctx, P_l, P_r, frames, edit=edit)
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(got, want), start=1):
        for q in range(len(frames)):
            where = f"sequence {q} frame {k}"
            if q == flat and k >= k_flat:
                continue
            if q == gone and k >= k_gone:
                r = a[q]
                assert r["status"] == capi.VO_MSEQ_RETIRED and r["n_features"] == 0, where
                m = r["mono"]
                assert all(m[key] == 0 for key in MONO_INTS), where
                assert not m["R"].any() and not m["t"].any() and len(r["ess_mask"]) == 0, where
                _, s_last, p_last = want[k_gone - 2]                     # frozen at its last frame, k_gone - 1
                assert np.array_equal(pa[q], p_last[q]), f"{where}: frozen frame_pose"
                _same_state(sa[q], s_last[q], f"{where}: frozen")
                continue
            _same(a[q], b[q], where)
            _same_state(sa[q], sb[q], where)
            assert np.array_equal(pa[q], pb[q]), f"{where}: frame_pose"
    # (got[k - 1] is frame k) both flat frames leave no valid match: the branch reports the reference's abort, R = I, and
    # frame_pose does not move
    for k in (k_flat, k_flat + 1):
        recs, _, poses = got[k - 1]
        r = recs[flat]
        assert r["status"] == capi.VO_OK and r["n_valid"] == 0, k
        assert r["mono"]["status"] == capi.VO_E_TOO_FEW_POINTS and np.array_equal(r["R"], np.eye(3)), k
        assert np.array_equal(poses[flat], got[k - 2][2][flat]), f"frame {k}: frame_pose moved"


def test_launches_per_submission_do_not_grow_with_the_sequence_count(built):
    from visual_odom_b200.capi import Context
    w, h = 320, 120
    base, fr = _drive(3, *DRIVES[0][1:], n=6, w=w, h=h)
    c = Context(0, max_features=1024)

    def per_submission(n, mono):
        c.mseq_begin([fr[0][0]] * n, [fr[0][1]] * n, base["P_l"], base["P_r"], mono_rotation=mono)
        for k in (1, 2):                      # captures the graphs of both buffer parities
            c.mseq_submit([fr[k][0]] * n, [fr[k][1]] * n); c.mseq_wait(want_points=False, mono=mono)
        l0 = c.kernel_launches()
        for k in range(3, 6):
            c.mseq_submit([fr[k][0]] * n, [fr[k][1]] * n); c.mseq_wait(want_points=False, mono=mono)
        return (c.kernel_launches() - l0) / 3

    one, sixteen, plain = per_submission(1, True), per_submission(16, True), per_submission(1, False)
    c.set_option("mono_rotation", 1)
    c.seq_begin(fr[0][0], fr[0][1], base["P_l"], base["P_r"])
    for k in (1, 2):
        c.seq_push(*fr[k], mono=True)
    l0 = c.kernel_launches()
    for k in range(3, 6):
        c.seq_push(*fr[k], mono=True)
    alone = (c.kernel_launches() - l0) / 3
    print(f"launches per submission: {one} with the flag (n_seq = 1 and 16), {alone} vo_seq_* with the option, {plain} without")
    assert one == sixteen == alone and one > plain > 0
    c.close()


def test_refusals_and_re_begins(built, ctx, sets, mono_runs):
    from visual_odom_b200 import capi
    from visual_odom_b200.capi import Context
    P_l, P_r, frames = sets["640x240"]
    n = len(frames)
    L = [fr[0][0] for fr in frames]; R = [fr[0][1] for fr in frames]

    def code(fn):
        with pytest.raises(capi.VoError) as e:
            fn()
        return e.value.code

    # vo_mseq_wait_mono on sequences begun without the flag; vo_mseq_wait on sequences begun with it
    ctx.mseq_begin(L, R, P_l, P_r)
    ctx.mseq_submit([fr[1][0] for fr in frames], [fr[1][1] for fr in frames])
    assert code(lambda: ctx.mseq_wait(mono=True)) == capi.VO_E_INVALID
    ctx.mseq_wait()
    ctx.mseq_begin(L, R, P_l, P_r, mono_rotation=True)
    ctx.mseq_submit([fr[1][0] for fr in frames], [fr[1][1] for fr in frames])
    plain = ctx.mseq_wait()
    for q in range(n):
        _same(plain[q], mono_runs["640x240"][0][0][q], f"vo_mseq_wait, sequence {q}", mono=False)
    # unknown flag bits, and the option with the flag
    lp, rp = (C.c_void_p * n)(*[x.ctypes.data for x in L]), (C.c_void_p * n)(*[x.ctypes.data for x in R])
    Pl = np.ascontiguousarray(P_l, np.float32); Pr = np.ascontiguousarray(P_r, np.float32)
    w, h = L[0].shape[1], L[0].shape[0]
    for flags in (2, capi.VO_MSEQ_MONO_ROTATION | 4, -1):
        assert ctx.lib.vo_mseq_begin_ex(ctx.h, n, w, h, Pl.ctypes.data, Pr.ctypes.data, lp, rp, w, 1, flags) == capi.VO_E_INVALID
    ctx.set_option("mono_rotation", 1)
    try:
        assert code(lambda: ctx.mseq_begin(L, R, P_l, P_r, mono_rotation=True)) == capi.VO_E_UNSUPPORTED
        assert code(lambda: ctx.mseq_begin(L, R, P_l, P_r)) == capi.VO_E_UNSUPPORTED
    finally:
        ctx.set_option("mono_rotation", 0)

    # flagged runs at n_seq = 2 and then 8 on one context (the mono scratch grows) equal fresh contexts; a vo_seq_* run
    # with the option afterwards equals a fresh context's
    two = frames[:2]
    eight = [frames[q % n] if q < n else frames[q % n][::-1] for q in range(8)]
    fresh = {}
    for key, fr in (("two", two), ("eight", eight)):
        f = Context(0, max_features=MAX_FEATURES)
        fresh[key] = _run_mseq(f, P_l, P_r, fr)
        f.close()
    f = Context(0, max_features=MAX_FEATURES)
    fresh["alone"] = _run_alone(f, P_l, P_r, frames[2])
    f.close()
    c = Context(0, max_features=MAX_FEATURES)
    try:
        _check_run(_run_mseq(c, P_l, P_r, two), fresh["two"], 2, "n_seq = 2: ")
        _check_run(_run_mseq(c, P_l, P_r, eight), fresh["eight"], 8, "n_seq = 8 after 2: ")
        for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(_run_alone(c, P_l, P_r, frames[2]), fresh["alone"]), start=1):
            _same(a, b, f"vo_seq_* after vo_mseq_*, frame {k}")
            _same_state(sa, sb, f"vo_seq_* after vo_mseq_*, frame {k}")
            assert np.array_equal(pa, pb), f"vo_seq_* after vo_mseq_*, frame {k}: frame_pose"
    finally:
        c.close()
