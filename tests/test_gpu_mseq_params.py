"""Tracking parameters per sequence of the multi-sequence mode (vo_mseq_params) and per unit of the batched mode
(vo_batch_params): every sequence / unit is bit for bit what a context created with its vo_params gives when it runs that
sequence alone (vo_seq_begin + vo_seq_push) or that unit alone (vo_frame_batch), in both buffer parities, pipelined, with
graphs off, with the mono_rotation branch, at several sizes, from device input, into device results, across retirement
and starts; the RANSAC bound is each unit's own count while the scratch keeps the context's stride; one sequence is
anchored to cv2 at its values; the context's own values set explicitly are no setting at all, at the same launch count;
and every refusal changes nothing."""
import numpy as np
import pytest

from visual_odom_b200 import synth
from test_gpu_mseq_calib import INTS, NF, SMALL, LARGE, _group, _alone, _run_mseq, _same

pytestmark = pytest.mark.gpu

CAP = 8192
# together these move every per-sequence field of vo_params off its default
SETTINGS = [
    dict(fast_threshold=12),
    dict(features_per_bucket=3, bucket_rows_divisor=6),
    dict(lk_max_iters=7, lk_epsilon=0.05, lk_min_eig=1e-2),
    dict(pnp_iterations=40, pnp_reproj_error=1.5, pnp_confidence=0.99),
    dict(refill_threshold=500, bucket_age_threshold=3, circ_threshold=1),
]


def _context(**prm):
    from visual_odom_b200.capi import Context
    return Context(0, max_features=prm.pop("max_features", CAP), **prm)


@pytest.fixture(scope="module")
def multi(built):
    c = _context()
    yield c
    c.close()


@pytest.fixture(scope="module")
def alone_ctx(built):
    """One context per setting, created with it."""
    cs = {i: _context(**s) for i, s in enumerate(SETTINGS)}
    yield cs
    for c in cs.values():
        c.close()


@pytest.fixture(scope="module", params=["small", "large"])
def group(request):
    spec = SMALL if request.param == "small" else LARGE
    n = len(spec[2])
    # the three large drives take settings 1, 2, 3 (the fields that depend on the image size most)
    idx = list(range(5)) if n == 5 else [1, 2, 3]
    return _group(spec) + (idx,)


@pytest.fixture(scope="module")
def small():
    return _group(SMALL) + (list(range(5)),)


def _set_slots(c, idx):
    c.mseq_params(0, [SETTINGS[i] if i is not None else None for i in idx])


def _reset_slots(c):
    from visual_odom_b200.capi import VO_MSEQ_MAX
    c.mseq_params(0, [None] * VO_MSEQ_MAX)


def _same_frames(run, alone, q, where):
    for k, ((recs, states, poses), (rec, st, pose)) in enumerate(zip(run, alone), start=1):
        _same(recs[q], rec, f"{where}: sequence {q} frame {k}")
        if states is not None:
            for name, a, b in zip(("points", "ages", "translation"), states[q], st):
                assert a.dtype == b.dtype and np.array_equal(a, b), f"{where}: sequence {q} frame {k}: carried {name}"
            assert np.array_equal(poses[q], pose), f"{where}: sequence {q} frame {k}: frame_pose"


@pytest.fixture(scope="module")
def small_alone(alone_ctx, small):
    P_l, P_r, frames, idx = small
    return [_alone(alone_ctx[i], P_l[q], P_r[q], frames[q]) for q, i in enumerate(idx)]


def test_each_sequence_equals_a_context_created_with_its_params(multi, alone_ctx, group):
    P_l, P_r, frames, idx = group
    _set_slots(multi, idx)
    try:
        run = _run_mseq(multi, P_l, P_r, frames)
    finally:
        _reset_slots(multi)
    default = _run_mseq(multi, P_l, P_r, frames)
    for q, i in enumerate(idx):
        alone = _alone(alone_ctx[i], P_l[q], P_r[q], frames[q])
        _same_frames(run, alone, q, f"setting {i}")
        assert alone[-1][0]["n_valid"] > 20
        # the setting matters: the same sequence at the context's values gives another run
        differs = any(any(not np.array_equal(np.asarray(a[0][q][key]), np.asarray(b[0][q][key])) for key in INTS + ("tvec", "l1"))
                      for a, b in zip(run, default))
        assert differs, f"setting {i} changes nothing on sequence {q}"


def test_pipelining_graphs_mono_and_retirement(multi, alone_ctx, small, small_alone):
    from visual_odom_b200 import capi
    P_l, P_r, frames, idx = small
    n = len(frames)
    _set_slots(multi, idx)
    try:
        # two submissions in flight, both buffer parities
        for k, ((a, _, _), alone_k) in enumerate(zip(_run_mseq(multi, P_l, P_r, frames, pipelined=True), zip(*small_alone)), start=1):
            for q in range(n):
                _same(a[q], alone_k[q][0], f"pipelined: sequence {q} frame {k}")
        # graphs off
        multi.set_option("graphs", 0)
        try:
            plain = _run_mseq(multi, P_l, P_r, frames)
        finally:
            multi.set_option("graphs", 1)
        for q in range(n):
            _same_frames(plain, small_alone[q], q, "graphs 0")
        # retirement leaves the others as they were
        gone, k_gone = 3, 2
        ret = _run_mseq(multi, P_l, P_r, frames, retire=(gone, k_gone))
        for q in range(n):
            if q == gone:
                assert all(ret[k - 1][0][q]["status"] == capi.VO_MSEQ_RETIRED for k in range(k_gone, NF))
                continue
            _same_frames(ret, small_alone[q], q, f"retired {gone}")
        # the mono_rotation branch
        mono = _run_mseq(multi, P_l, P_r, frames, mono=True)
    finally:
        _reset_slots(multi)
    for q, i in enumerate(idx):
        alone = _alone(alone_ctx[i], P_l[q], P_r[q], frames[q], mono=True)
        _same_frames(mono, alone, q, "mono")
        for k, ((recs, _, _), (rec, _, _)) in enumerate(zip(mono, alone), start=1):
            for key in ("status", "n_inliers", "ransac_iters", "n_good"):
                assert recs[q]["mono"][key] == rec["mono"][key], f"mono: sequence {q} frame {k}: {key}"
            assert np.array_equal(recs[q]["mono"]["R"], rec["mono"]["R"]) and np.array_equal(recs[q]["ess_mask"], rec["ess_mask"])


def test_sequences_of_several_sizes(multi, alone_ctx):
    """vo_mseq_begin_sized: two 640x240 and two 1241x376 drives, each at its own setting."""
    Ps, Pr_s, fs = _group(SMALL)
    Pl_l, Pr_l, fl = _group(LARGE)
    P_l = np.stack([Ps[0], Pl_l[0], Ps[1], Pl_l[1]]); P_r = np.stack([Pr_s[0], Pr_l[0], Pr_s[1], Pr_l[1]])
    frames = [fs[0], fl[0], fs[1], fl[1]]
    idx = [1, 4, 2, 0]
    _set_slots(multi, idx)
    try:
        run = _run_mseq(multi, P_l, P_r, frames)
    finally:
        _reset_slots(multi)
    for q, i in enumerate(idx):
        _same_frames(run, _alone(alone_ctx[i], P_l[q], P_r[q], frames[q]), q, f"sized, setting {i}")


def test_device_input_and_device_results(multi, alone_ctx, small, small_alone):
    torch = pytest.importorskip("torch")
    from visual_odom_b200 import capi
    P_l, P_r, frames, idx = small
    n = len(frames)
    dev = [[(torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda()) for l, r in fr] for fr in frames]
    _set_slots(multi, idx)
    try:
        # device input, host waits
        multi.mseq_begin_device([d[0][0] for d in dev], [d[0][1] for d in dev], P_l, P_r)
        for k in range(1, NF):
            multi.mseq_submit_device([d[k][0] for d in dev], [d[k][1] for d in dev])
            recs = multi.mseq_wait()
            for q in range(n):
                _same(recs[q], small_alone[q][k - 1][0], f"device input: sequence {q} frame {k}")
        # device results: records, frame_pose, the point lists, points3D and inliers
        multi.mseq_begin_device([d[0][0] for d in dev], [d[0][1] for d in dev], P_l, P_r, device_results=True)
        got = []
        for k in range(1, NF):
            multi.mseq_submit_device([d[k][0] for d in dev], [d[k][1] for d in dev])
            out = multi.mseq_wait_device(pts_cap=CAP)
            torch.cuda.synchronize()
            got.append({key: v.cpu().numpy() for key, v in out.items() if hasattr(v, "cpu")})
    finally:
        _reset_slots(multi)
    for q, i in enumerate(idx):
        c = alone_ctx[i]
        c.mseq_begin_device([dev[q][0][0]], [dev[q][0][1]], P_l[q], P_r[q], device_results=True)
        for k in range(1, NF):
            c.mseq_submit_device([dev[q][k][0]], [dev[q][k][1]])
            out = c.mseq_wait_device(pts_cap=CAP)
            torch.cuda.synchronize()
            ref = {key: v.cpu().numpy() for key, v in out.items() if hasattr(v, "cpu")}
            g = got[k - 1]
            where = f"device results: sequence {q} frame {k}"
            assert g["status"][q] == ref["status"][0] == capi.VO_OK, where
            assert np.array_equal(g["records"][q].view(np.uint8), ref["records"][0].view(np.uint8)), where
            assert np.array_equal(g["frame_pose"][q], ref["frame_pose"][0]), where
            nv, ni = int(ref["counts"][0][3]), int(ref["counts"][0][4])
            assert np.array_equal(g["pts4"][q][:, :nv], ref["pts4"][0][:, :nv]), where
            assert np.array_equal(g["points3d"][q][:nv], ref["points3d"][0][:nv]), where
            assert np.array_equal(g["inliers"][q][:ni], ref["inliers"][0][:ni]), where
            assert np.array_equal(g["frame_pose"][q], small_alone[q][k - 1][2]), where


def test_a_start_takes_the_slots_new_params_while_the_old_frame_is_in_flight(multi, alone_ctx, small, small_alone):
    """Slot 2 runs setting 2; with its frame 1 in flight it is set to setting 0 and a new sequence (drive 4) starts in it.
    The old sequence's last frame keeps setting 2, the new sequence equals a context created with setting 0."""
    from visual_odom_b200 import capi
    P_l, P_r, frames, idx = small
    n = len(frames)
    _set_slots(multi, idx)
    new = 4
    try:
        multi.mseq_begin([f[0][0] for f in frames], [f[0][1] for f in frames], P_l, P_r)
        def submit(k, slot2, start=None):          # frame k of the others (None: retired), slot2 = slot 2's pair
            ps = [(frames[q][k] if k is not None else (None, None)) if q != 2 else slot2 for q in range(n)]
            multi.mseq_submit([p[0] for p in ps], [p[1] for p in ps], start=start)

        submit(1, frames[2][1])
        multi.mseq_params(2, [SETTINGS[0]])                         # frame 1 is in flight
        submit(2, frames[new][0], start={2: (P_l[new], P_r[new])})
        r1 = multi.mseq_wait()
        submit(3, frames[new][1])
        r2 = multi.mseq_wait()
        submit(4, frames[new][2])
        r3 = multi.mseq_wait()
        submit(None, frames[new][3])
        r4 = multi.mseq_wait()
        r5 = multi.mseq_wait()
    finally:
        _reset_slots(multi)
    _same(r1[2], small_alone[2][0][0], "old sequence, frame 1")
    assert r2[2]["status"] == capi.VO_MSEQ_STARTED
    fresh = _alone(alone_ctx[0], P_l[new], P_r[new], frames[new])
    _same(r3[2], fresh[0][0], "new sequence, frame 1")
    _same(r4[2], fresh[1][0], "new sequence, frame 2")
    _same(r5[2], fresh[2][0], "new sequence, frame 3")
    for q in (0, 1, 3, 4):
        for k, r in enumerate((r1, r2, r3, r4), start=1):
            _same(r[q], small_alone[q][k - 1][0], f"sequence {q} frame {k}")


def test_the_pnp_bound_is_each_units_own_count_and_the_stride_the_contexts(built):
    """In a context of 500 RANSAC iterations, units and sequences at 1, 31, 32, 33, 127, 128, 129 and 0 iterations give
    what contexts created with those counts give, inliers included (a tight reprojection threshold keeps RANSAC long)."""
    counts = [1, 31, 32, 33, 127, 128, 129, 0]
    base = dict(pnp_reproj_error=0.05)
    units, P_l, P_r = _units()
    c = _context(pnp_iterations=500, **base)
    c.set_option("batch_outputs", 1)
    c.batch_configure(BW, BH, len(counts), P_l[0], P_r[0])
    c.batch_calibrate(0, P_l[:len(counts)], P_r[:len(counts)])
    c.batch_params(0, [dict(pnp_iterations=m, **base) for m in counts])
    keep = _submit(c, units[:len(counts)], 0)
    got = _collect(c, 0, len(counts))
    iters = []
    for i, m in enumerate(counts):
        a = _context(pnp_iterations=m, **base)
        a.set_option("batch_outputs", 1)
        a.batch_configure(BW, BH, len(counts), P_l[i], P_r[i])
        keep = _submit(a, units[:len(counts)], 0)
        ref = _collect(a, 0, len(counts))[i]
        a.close()
        _same_unit(got[i], ref, f"unit at {m} iterations")
        assert got[i][0]["ransac_iters"] <= max(m, 1)
        iters.append(got[i][0]["ransac_iters"])
    assert len(set(iters)) >= 3, iters                 # the bounds are reached
    # the same counts per sequence (the five small drives, three of them twice)
    Pl, Pr, frames = _group(SMALL)
    sel = [q % 5 for q in range(len(counts))]
    c.mseq_params(0, [dict(pnp_iterations=m, **base) for m in counts])
    run = _run_mseq(c, Pl[sel], Pr[sel], [frames[q] for q in sel])
    c.close()
    for q, m in enumerate(counts):
        a = _context(pnp_iterations=m, **base)
        alone = _alone(a, Pl[sel[q]], Pr[sel[q]], frames[sel[q]])
        a.close()
        _same_frames(run, alone, q, f"sequence at {m} iterations")


def test_a_sequence_at_its_params_matches_the_reference_loop(multi, small):
    """Sequence 1 (three features per bucket, bucket size rows / 6) frame by frame against the reference loop restated
    with those values over cv2 (test_gpu_bucketing's glue)."""
    pytest.importorskip("cv2")
    from test_gpu_bucketing import _oracle, _check
    P_l, P_r, frames, idx = small
    _set_slots(multi, idx)
    try:
        run = _run_mseq(multi, P_l, P_r, frames)
    finally:
        _reset_slots(multi)
    ref = _oracle(P_l[1], P_r[1], frames[1], dict(SETTINGS[1]))
    for k, ((recs, states, _), r) in enumerate(zip(run, ref), start=1):
        _check(recs[1], states[1], r, f"frame {k}")


def test_the_contexts_own_values_are_no_setting_at_the_same_launch_count(built, small):
    P_l, P_r, frames, _ = small
    n = len(frames)
    c = _context()

    def launches():
        c.mseq_begin([f[0][0] for f in frames], [f[0][1] for f in frames], P_l, P_r)
        out = []
        for k in (1, 2):                                       # captures both buffer parities
            c.mseq_submit(*zip(*[f[k] for f in frames])); out.append(c.mseq_wait())
        l0 = c.kernel_launches()
        for k in (3, 4):
            c.mseq_submit(*zip(*[f[k] for f in frames])); out.append(c.mseq_wait())
        return out, (c.kernel_launches() - l0) / 2

    plain, n_plain = launches()
    c.mseq_params(0, [{} for _ in range(n)])                   # explicitly the context's values
    explicit, n_explicit = launches()
    c.mseq_params(0, [SETTINGS[q] for q in range(n)])
    _, n_set = launches()
    c.close()
    assert n_plain == n_explicit == n_set == 30
    for k, (a, b) in enumerate(zip(explicit, plain), start=1):
        for q in range(n):
            _same(a[q], b[q], f"explicit: sequence {q} frame {k}")


# ---- batched mode ----------------------------------------------------------------------------------------------------
BW, BH = 640, 240
BATCH_SETTINGS = SETTINGS + [dict(), dict(fast_threshold=30, lk_max_iters=15), dict(circ_threshold=2, pnp_reproj_error=0.8)]


def _units():
    cals = [d[3] for d in SMALL[2]] * 2
    units, P_l, P_r = [], [], []
    for i, cal in enumerate(cals[:8]):
        u = synth.stereo_unit(BW, BH, 100 + i, cal=cal)
        units.append(dict(l0=u["l0"], r0=u["r0"], l1=u["l1"], r1=u["r1"], n_select=1500))
        P_l.append(u["P_l"]); P_r.append(u["P_r"])
    return units, np.stack(P_l), np.stack(P_r)


def _submit(c, units, slot0):
    arr, keep, pitch = c.make_units(units)
    c.batch_submit(arr, slot0, pitch)
    return keep


def _collect(c, slot0, n):
    recs = c.batch_wait(slot0, n)
    return [(r, c.batch_outputs(slot0 + i, r)) for i, r in enumerate(recs)]


def _same_unit(a, b, where):
    (ra, oa), (rb, ob) = a, b
    _same(ra, rb, where, keys=("rvec", "tvec", "R"))
    for k in ("l0", "r0", "l1", "r1", "kept_idx", "X", "inliers"):
        assert np.array_equal(oa[k], ob[k]), f"{where}: {k}"


def test_batch_units_with_their_own_params_equal_units_run_alone(built):
    """On-GPU detection at each unit's FAST threshold, its LK criteria, validity threshold and PnP settings;
    vo_batch_configure resets every unit to the context's."""
    units, P_l, P_r = _units()
    B = len(units)
    c = _context()
    c.set_option("batch_outputs", 1)
    c.batch_configure(BW, BH, B, P_l[0], P_r[0])
    c.batch_calibrate(0, P_l, P_r)
    keep = _submit(c, units, 0)
    default = _collect(c, 0, B)
    c.batch_params(0, BATCH_SETTINGS)
    keep = _submit(c, units, 0)
    got = _collect(c, 0, B)
    for i, s in enumerate(BATCH_SETTINGS):
        a = _context(**s)
        a.set_option("batch_outputs", 1)
        a.batch_configure(BW, BH, B, P_l[0], P_r[0])
        a.batch_calibrate(0, P_l, P_r)
        keep = _submit(a, units, 0)
        ref = _collect(a, 0, B)[i]
        # vo_frame_batch of the same units
        arr, keep2, pitch = a.make_units(units)
        fb = a.frame_batch(arr, pitch)[i]
        a.close()
        _same_unit(got[i], ref, f"unit {i}")
        _same(got[i][0], fb, f"unit {i} against vo_frame_batch", keys=("rvec", "tvec", "R"))
        changed = any(got[i][0][k] != default[i][0][k] for k in INTS) or not np.array_equal(got[i][0]["tvec"], default[i][0]["tvec"])
        # the batched path reads every field but the four bookkeeping ones, which it ignores
        assert changed == bool(set(s) - {"refill_threshold", "bucket_rows_divisor", "features_per_bucket", "bucket_age_threshold"}), \
            f"unit {i}: {s}"
    c.batch_configure(BW, BH, B, P_l[0], P_r[0])
    c.batch_calibrate(0, P_l, P_r)
    keep = _submit(c, units, 0)
    after = _collect(c, 0, B)
    for i in range(B):
        _same_unit(after[i], default[i], f"unit {i} after vo_batch_configure")
    c.close()


def test_refusals_change_nothing(built, small, alone_ctx):
    from visual_odom_b200 import capi
    P_l, P_r, frames, idx = small
    n = len(frames)
    c = _context(pnp_iterations=200)

    def code(fn):
        with pytest.raises(capi.VoError) as e:
            fn()
        return e.value.code

    # field values, with vo_create's codes and messages
    bad = [(dict(fast_threshold=256), capi.VO_E_INVALID, "fast_threshold=256 outside [0,255]"),
           (dict(pnp_confidence=1.0), capi.VO_E_INVALID, "pnp_confidence=1 outside (0,1)"),
           (dict(bucket_rows_divisor=0), capi.VO_E_INVALID, "bucket_rows_divisor=0"),
           (dict(features_per_bucket=0), capi.VO_E_INVALID, "features_per_bucket=0"),
           (dict(lk_win=15), capi.VO_E_UNSUPPORTED, "lk_win=15"),
           (dict(lk_max_level=2), capi.VO_E_UNSUPPORTED, "lk_max_level=2"),
           (dict(fast_nonmax=0), capi.VO_E_UNSUPPORTED, "fast_nonmax=0"),
           (dict(pnp_iterations=201), capi.VO_E_CAPACITY, "pnp_iterations=201")]
    for prm, rc, msg in bad:
        with pytest.raises(capi.VoError) as e:
            c.mseq_params(0, [None, prm])
        assert e.value.code == rc and msg in str(e.value) and "slot 1" in str(e.value), (prm, str(e.value))
    c.mseq_params(0, [dict(pnp_iterations=200), dict(pnp_iterations=-5)])      # at the context's count, and <= 0: accepted
    arr = (capi.VoParams * 1)(c.params_with())
    for first, m in ((-1, 1), (capi.VO_MSEQ_MAX, 1), (capi.VO_MSEQ_MAX - 1, 2), (0, 0)):
        assert c.lib.vo_mseq_params(c.h, first, m, arr) == capi.VO_E_INVALID, (first, m)
    assert c.lib.vo_mseq_params(c.h, 0, capi.VO_MSEQ_MAX, None) == capi.VO_OK       # NULL: the context's again
    # per-sequence capacity at begin, open and start: a bound above max_features, a zero bucket size
    small_cap = _context(max_features=2048)
    small_cap.mseq_params(1, [dict(features_per_bucket=20)])
    with pytest.raises(capi.VoError) as e:
        small_cap.mseq_begin([f[0][0] for f in frames[:2]], [f[0][1] for f in frames[:2]], P_l[:2], P_r[:2])
    assert e.value.code == capi.VO_E_CAPACITY and "sequence 1" in str(e.value)
    assert code(lambda: small_cap.mseq_open(2, BW, BH)) == capi.VO_E_CAPACITY
    small_cap.mseq_params(1, [dict(bucket_rows_divisor=400)])
    assert code(lambda: small_cap.mseq_open(2, BW, BH)) == capi.VO_E_UNSUPPORTED
    small_cap.mseq_params(1, [None])
    small_cap.mseq_open(2, BW, BH)
    small_cap.mseq_params(1, [dict(features_per_bucket=20)])
    both = dict(start={0: (P_l[0], P_r[0]), 1: (P_l[1], P_r[1])})
    first_pairs = ([frames[0][0][0], frames[1][0][0]], [frames[0][0][1], frames[1][0][1]])
    assert code(lambda: small_cap.mseq_submit(*first_pairs, **both)) == capi.VO_E_CAPACITY
    small_cap.mseq_params(1, [None])
    small_cap.mseq_submit(*first_pairs, **both)                 # the refused start changed nothing
    assert [r["status"] for r in small_cap.mseq_wait()] == [capi.VO_MSEQ_STARTED] * 2
    small_cap.close()
    # batched: ranges, fields, a submission in flight
    units, Pl, Pr = _units()
    c.set_option("batch_outputs", 1)
    c.batch_configure(BW, BH, 8, Pl[0], Pr[0])
    assert code(lambda: c.batch_params(7, [{}, {}])) == capi.VO_E_INVALID
    assert code(lambda: c.batch_params(-1, [{}])) == capi.VO_E_INVALID
    assert code(lambda: c.batch_params(0, [dict(fast_threshold=-1)])) == capi.VO_E_INVALID
    assert code(lambda: c.batch_params(0, [dict(pnp_iterations=201)])) == capi.VO_E_CAPACITY
    assert code(lambda: c.batch_params(0, [dict(lk_max_level=4)])) == capi.VO_E_UNSUPPORTED
    keep = _submit(c, units, 0)
    assert code(lambda: c.batch_params(0, [dict(fast_threshold=12)])) == capi.VO_E_INVALID
    first = _collect(c, 0, 8)
    keep = _submit(c, units, 0)
    again = _collect(c, 0, 8)
    for i in range(8):
        _same_unit(again[i], first[i], f"unit {i} after the refusals")
    c.close()
    # and a multi-sequence run after refused calls equals a fresh context
    fresh = _context(pnp_iterations=200)
    f = _run_mseq(fresh, P_l, P_r, frames)
    fresh.close()
    c2 = _context(pnp_iterations=200)
    for prm, _, _ in bad:
        with pytest.raises(capi.VoError):
            c2.mseq_params(0, [prm] * n)
    g = _run_mseq(c2, P_l, P_r, frames)
    c2.close()
    for q in range(n):
        _same_frames(g, [(r[0][q], r[1][q], r[2][q]) for r in f], q, "after refusals")
