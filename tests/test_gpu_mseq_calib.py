"""One calibration per sequence of the multi-sequence mode (vo_mseq_begin_calib) and per unit of the batched mode
(vo_batch_calibrate): every sequence / unit is bit for bit what it gives when run alone with its own matrices, in both
buffer parities, with the mono_rotation branch, under pipelining, reordering, retirement and graphs on or off; one
sequence and one unit are anchored to cv2 with their own P; one calibration repeated is vo_mseq_begin_ex exactly, at the
same launch count; and every refusal leaves the context usable."""
import ctypes as C

import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

K0 = synth.KITTI00
NF = 5                      # frames 0 .. 4: four submissions, both buffer parities twice


def _cal(sx=1.0, sy=1.0, dcx=0.0, dcy=0.0, sb=1.0):
    return dict(fx=K0["fx"] * sx, fy=K0["fy"] * sy, cx=K0["cx"] + dcx, cy=K0["cy"] + dcy, bf=K0["bf"] * sb)


# (seed, per-frame rotation, per-frame translation, calibration): five drives at 640x240, three at 1241x376
SMALL = (640, 240, [
    (31, (0.001, -0.004, 0.0005), (0.01, -0.003, -0.2), _cal()),
    (7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25), _cal(0.9, 0.9)),
    (13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15), _cal(1.1, 1.1, 25.0, -15.0)),
    (42, (0.003, -0.001, 0.0005), (0.015, 0.0, -0.3), _cal(1.0, 1.0, -40.0, 20.0, 1.15)),
    (5, (-0.001, -0.002, 0.001), (0.0, -0.005, -0.18), _cal(0.95, 1.05, 10.0, 30.0, 0.85)),
])
LARGE = (1241, 376, [
    (3, (0.001, 0.002, 0.0), (0.01, 0.0, -0.22), _cal(1.1, 1.1, 0.0, 0.0, 0.85)),
    (11, (-0.002, -0.001, 0.0005), (0.0, 0.003, -0.2), _cal(0.9, 0.9, -30.0, 12.0)),
    (19, (0.0, -0.003, 0.001), (-0.01, 0.0, -0.26), _cal(1.0, 1.0, 35.0, -20.0, 1.15)),
])
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
ARRAYS = ("rvec", "tvec", "R", "l0", "r0", "l1", "r1")


def _group(spec):
    w, h, drives = spec
    P_l, P_r, frames = [], [], []
    for seed, r, t, cal in drives:
        base = synth.stereo_unit(w, h, seed, cal=cal)
        fr = [(base["l0"], base["r0"])]
        for k in range(1, NF):
            u = synth.stereo_unit(w, h, seed, cal=cal, rvec=np.array(r) * k, tvec=np.array(t) * k)
            fr.append((u["l1"], u["r1"]))
        P_l.append(base["P_l"]); P_r.append(base["P_r"]); frames.append(fr)
    return np.stack(P_l), np.stack(P_r), frames


@pytest.fixture(scope="module", params=["small", "large"])
def group(request):
    return _group(SMALL if request.param == "small" else LARGE)


@pytest.fixture(scope="module")
def small():
    return _group(SMALL)


def _same(a, b, where, keys=ARRAYS):
    for k in INTS:
        assert a[k] == b[k], f"{where}: {k} {a[k]} != {b[k]}"
    for k in keys:
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), f"{where}: {k}"


def _run_mseq(ctx, P_l, P_r, frames, pipelined=False, mono=False, retire=None):
    """Per frame: (records, [state of q], [pose of q]); state / pose only for submit-then-wait runs.  retire = (q, k):
    sequence q gets a NULL pair from frame k on."""
    n = len(frames)
    ctx.mseq_begin([f[0][0] for f in frames], [f[0][1] for f in frames], P_l, P_r, mono_rotation=mono)

    def submit(k):
        ps = [(None, None) if retire and q == retire[0] and k >= retire[1] else frames[q][k] for q in range(n)]
        ctx.mseq_submit([p[0] for p in ps], [p[1] for p in ps])

    out = []
    if pipelined:
        submit(1)
        for k in range(1, NF):
            if k + 1 < NF:
                submit(k + 1)
            out.append((ctx.mseq_wait(mono=mono), None, None))
        return out
    for k in range(1, NF):
        submit(k)
        recs = ctx.mseq_wait(mono=mono)
        out.append((recs, [ctx.mseq_state(q) for q in range(n)], [ctx.mseq_pose(q) for q in range(n)]))
    return out


def _alone(ctx, P_l, P_r, fr, mono=False):
    """vo_seq_begin / vo_seq_push of one sequence with its own matrices: per frame (record, state, pose)."""
    ctx.set_option("mono_rotation", 1 if mono else 0)
    try:
        ctx.seq_begin(fr[0][0], fr[0][1], P_l, P_r)
        out = []
        for k in range(1, NF):
            rec = ctx.seq_push(*fr[k], mono=mono)
            out.append((rec, ctx.seq_state(), ctx.seq_pose()))
        return out
    finally:
        ctx.set_option("mono_rotation", 0)


def _check_against_alone(ctx, P_l, P_r, frames, run, mono=False):
    from visual_odom_b200 import capi
    for q, fr in enumerate(frames):
        alone = _alone(ctx, P_l[q], P_r[q], fr, mono)
        for k, ((recs, states, poses), (rec, st, pose)) in enumerate(zip(run, alone), start=1):
            assert recs[q]["status"] == capi.VO_OK
            _same(recs[q], rec, f"sequence {q} frame {k}")
            if mono:
                for key in ("status", "n_inliers", "ransac_iters", "n_good"):
                    assert recs[q]["mono"][key] == rec["mono"][key], f"sequence {q} frame {k}: mono {key}"
                for key in ("R", "t"):
                    assert np.array_equal(recs[q]["mono"][key], rec["mono"][key]), f"sequence {q} frame {k}: mono {key}"
                assert np.array_equal(recs[q]["ess_mask"], rec["ess_mask"]), f"sequence {q} frame {k}: essential mask"
            for name, a, b in zip(("points", "ages", "translation"), states[q], st):
                assert a.dtype == b.dtype and np.array_equal(a, b), f"sequence {q} frame {k}: carried {name}"
            assert np.array_equal(poses[q], pose), f"sequence {q} frame {k}: frame_pose"
        assert alone[-1][0]["n_valid"] > 50 and alone[-1][0]["n_inliers"] > 20
    # the calibrations differ enough to matter: sequence 0's frames under sequence 1's matrices give another pose
    other = _alone(ctx, P_l[1], P_r[1], frames[0])
    assert not np.array_equal(other[-1][0]["tvec"], run[-1][0][0]["tvec"])


def test_each_sequence_is_bit_identical_to_running_it_alone_with_its_calibration(ctx, group):
    P_l, P_r, frames = group
    assert len({p.tobytes() for p in P_l}) == len(frames) and len({p.tobytes() for p in P_r}) == len(frames)
    _check_against_alone(ctx, P_l, P_r, frames, _run_mseq(ctx, P_l, P_r, frames))


def test_mono_branch_is_bit_identical_to_running_it_alone_with_its_calibration(ctx, small):
    P_l, P_r, frames = small
    _check_against_alone(ctx, P_l, P_r, frames, _run_mseq(ctx, P_l, P_r, frames, mono=True), mono=True)


def test_a_sequence_other_than_the_first_matches_the_reference_path(ctx, small):
    """Sequence 2 frame by frame against cv2 through the reference's glue (oracle/ref_path.py) with ITS matrices."""
    pytest.importorskip("cv2")
    from oracle import ref_path
    P_l, P_r, frames = small
    run = _run_mseq(ctx, P_l, P_r, frames)
    q = 2
    fr = frames[q]
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    for k in range(1, NF):
        (l0, r0), (l1, r1) = fr[k - 1], fr[k]
        recs, states, poses = run[k - 1]
        got = recs[q]
        pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend="cv2")
        X = ref_path.triangulate(P_l[q], P_r[q], pL0, pR0, "cv2")
        R, translation, inl, rvec = ref_path.tracking_frame2frame(P_l[q], pL0, pL1, X, translation, "cv2")
        assert got["n_features"] == len(info["bucketed"]) and got["n_tracked"] == len(info["kept_idx"])
        assert got["n_valid"] == len(pL0)
        for name, ref in (("l0", pL0), ("r0", pR0), ("l1", pL1), ("r1", pR1)):
            assert np.array_equal(got[name], ref), f"frame {k}: {name}"
        assert got["n_inliers"] == len(inl), f"frame {k}: inlier count"
        assert np.linalg.norm(got["R"] - R) / np.linalg.norm(R) <= 1e-4
        assert np.linalg.norm(got["tvec"] - translation) / np.linalg.norm(translation) <= 1e-4
        frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
        assert np.abs(poses[q] - frame_pose).max() <= 1e-6 * max(1.0, np.abs(frame_pose).max()), f"frame {k}: frame_pose"
        pts, ages, _ = states[q]
        assert np.array_equal(pts, fs.points) and np.array_equal(ages, fs.ages), f"frame {k}: carried FeatureSet"


def test_indexing_order_pipelining_graphs_and_retirement(ctx, small):
    P_l, P_r, frames = small
    n = len(frames)
    ref = _run_mseq(ctx, P_l, P_r, frames)
    # reversing the sequences (with their calibrations) reverses the results
    rev = _run_mseq(ctx, P_l[::-1], P_r[::-1], frames[::-1])
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(rev, ref), start=1):
        for q in range(n):
            _same(a[n - 1 - q], b[q], f"reversed: sequence {q} frame {k}")
            assert np.array_equal(pa[n - 1 - q], pb[q])
            assert all(np.array_equal(x, y) for x, y in zip(sa[n - 1 - q], sb[q]))
    # two submissions in flight = submit-then-wait
    for k, ((a, _, _), (b, _, _)) in enumerate(zip(_run_mseq(ctx, P_l, P_r, frames, pipelined=True), ref), start=1):
        for q in range(n):
            _same(a[q], b[q], f"pipelined: sequence {q} frame {k}")
    # graphs off = graphs on
    ctx.set_option("graphs", 0)
    try:
        plain = _run_mseq(ctx, P_l, P_r, frames)
    finally:
        ctx.set_option("graphs", 1)
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(plain, ref), start=1):
        for q in range(n):
            _same(a[q], b[q], f"graphs 0: sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q])
    # a retired sequence leaves the others bit-identical
    from visual_odom_b200 import capi
    gone, k_gone = 1, 2
    ret = _run_mseq(ctx, P_l, P_r, frames, retire=(gone, k_gone))
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(ret, ref), start=1):
        for q in range(n):
            if q == gone and k >= k_gone:
                assert a[q]["status"] == capi.VO_MSEQ_RETIRED
                continue
            _same(a[q], b[q], f"retired {gone}: sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q]) and all(np.array_equal(x, y) for x, y in zip(sa[q], sb[q]))


def test_one_calibration_repeated_is_begin_ex_bit_for_bit_and_at_the_same_launch_count(ctx, small, built):
    P_l, P_r, frames = small
    n = len(frames)
    one = _run_mseq(ctx, P_l[0], P_r[0], frames)                                   # vo_mseq_begin_ex
    rep = _run_mseq(ctx, np.stack([P_l[0]] * n), np.stack([P_r[0]] * n), frames)    # vo_mseq_begin_calib
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(rep, one), start=1):
        for q in range(n):
            _same(a[q], b[q], f"sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q]) and all(np.array_equal(x, y) for x, y in zip(sa[q], sb[q]))

    from visual_odom_b200.capi import Context
    w, h = 320, 120
    fr = [(synth.stereo_unit(w, h, 3)["l0"], synth.stereo_unit(w, h, 3)["r0"])]
    for k in range(1, 6):
        u = synth.stereo_unit(w, h, 3, rvec=np.array((0.001, -0.004, 0.0005)) * k, tvec=np.array((0.01, -0.003, -0.2)) * k)
        fr.append((u["l1"], u["r1"]))
    Pl0, Pr0 = synth.proj_matrices()
    c = Context(0, max_features=1024)

    def per_submission(m, calib):
        Pl = np.stack([synth.proj_matrices(_cal(1 + 0.01 * q))[0] for q in range(m)]) if calib else Pl0
        Pr = np.stack([synth.proj_matrices(_cal(1 + 0.01 * q))[1] for q in range(m)]) if calib else Pr0
        c.mseq_begin([fr[0][0]] * m, [fr[0][1]] * m, Pl, Pr)
        for k in (1, 2):                      # captures the graphs of both buffer parities
            c.mseq_submit([fr[k][0]] * m, [fr[k][1]] * m); c.mseq_wait(want_points=False)
        l0 = c.kernel_launches()
        for k in range(3, 6):
            c.mseq_submit([fr[k][0]] * m, [fr[k][1]] * m); c.mseq_wait(want_points=False)
        return (c.kernel_launches() - l0) / 3

    calib1, calib16, ex16 = per_submission(1, True), per_submission(16, True), per_submission(16, False)
    c.seq_begin(fr[0][0], fr[0][1], Pl0, Pr0)
    for k in (1, 2):
        c.seq_push(*fr[k])
    l0 = c.kernel_launches()
    for k in range(3, 6):
        c.seq_push(*fr[k])
    alone = (c.kernel_launches() - l0) / 3
    c.close()
    assert calib1 == calib16 == ex16 == alone and alone > 0


# ---- batched mode ----------------------------------------------------------------------------------------------------
B = 8
BW, BH = 640, 240


@pytest.fixture(scope="module")
def batch_units():
    """Eight units at 640x240, each rendered with its own calibration."""
    cals = [d[3] for d in SMALL[2]] + [_cal(1.05, 1.05, -10.0, 5.0, 0.9), _cal(0.92, 0.92, 15.0, -10.0, 1.1),
                                        _cal(1.0, 1.0, 50.0, 0.0, 1.05)]
    units, P_l, P_r = [], [], []
    for i, cal in enumerate(cals):
        u = synth.stereo_unit(BW, BH, 100 + i, cal=cal)
        units.append(dict(l0=u["l0"], r0=u["r0"], l1=u["l1"], r1=u["r1"], n_select=1500))
        P_l.append(u["P_l"]); P_r.append(u["P_r"])
    return units, np.stack(P_l), np.stack(P_r)


def _batch_context():
    from visual_odom_b200.capi import Context
    c = Context(0, max_features=4096)
    c.set_option("batch_outputs", 1)
    return c


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


@pytest.fixture(scope="module")
def batch_alone(batch_units):
    """unit i of a context configured with calibration i alone (every unit submitted, unit i kept)."""
    units, P_l, P_r = batch_units
    c = _batch_context()
    out = []
    for i in range(B):
        c.batch_configure(BW, BH, B, P_l[i], P_r[i])
        keep = _submit(c, units, 0)
        res = _collect(c, 0, B)
        del keep
        out.append(res[i])
    c.close()
    return out


def test_batch_units_with_their_own_calibrations_equal_units_run_alone(batch_units, batch_alone):
    units, P_l, P_r = batch_units
    c = _batch_context()
    c.batch_configure(BW, BH, B, P_l[0], P_r[0])
    c.batch_calibrate(0, P_l, P_r)
    keep = _submit(c, units, 0)
    got = _collect(c, 0, B)
    for i in range(B):
        _same_unit(got[i], batch_alone[i], f"unit {i}")
        assert got[i][0]["n_inliers"] > 20
    # the same units through vo_batch_run (one range replayed as a graph on the context's stream, and as two lanes)
    for streams in (1, 2):
        c.set_option("batch_streams", streams)
        arr, keep2, pitch = c.make_units(units)
        c.batch_upload(arr, pitch)
        c.batch_run()
        for i, r in enumerate(c.batch_download(B)):
            _same(r, batch_alone[i][0], f"vo_batch_run, {streams} stream(s): unit {i}", keys=("rvec", "tvec", "R"))
    c.close()


def test_two_slot_ranges_with_different_calibrations_in_flight(batch_units, batch_alone):
    units, P_l, P_r = batch_units
    c = _batch_context()
    c.batch_configure(BW, BH, 2 * B, P_l[0], P_r[0])
    c.batch_calibrate(0, P_l, P_r)
    c.batch_calibrate(B, P_l[::-1], P_r[::-1])
    k0 = _submit(c, units, 0)
    k1 = _submit(c, units[::-1], B)
    a = _collect(c, 0, B)
    b = _collect(c, B, B)
    for i in range(B):
        _same_unit(a[i], batch_alone[i], f"range 0 unit {i}")
        _same_unit(b[i], batch_alone[B - 1 - i], f"range 1 unit {i}")
    c.close()


def test_a_batch_unit_matches_cv2_with_its_calibration(batch_units, batch_alone):
    """Unit 3's triangulation and pose against cv2 with ITS P, from the point lists the unit returned."""
    pytest.importorskip("cv2")
    from oracle import ref_path
    units, P_l, P_r = batch_units
    c = _batch_context()
    c.batch_configure(BW, BH, B, P_l[0], P_r[0])
    c.batch_calibrate(0, P_l, P_r)
    keep = _submit(c, units, 0)
    r, o = _collect(c, 0, B)[3]
    c.close()
    X = ref_path.triangulate(P_l[3], P_r[3], o["l0"], o["r0"], "cv2")
    rel = np.linalg.norm(o["X"] - X, axis=1) / np.maximum(np.linalg.norm(X, axis=1), 1e-6)
    assert np.mean(rel <= 1e-4) >= 0.99, f"median relative error {np.median(rel)}"
    R, t, inl, rvec = ref_path.tracking_frame2frame(P_l[3], o["l0"], o["l1"], X, np.zeros(3), "cv2")
    assert r["n_inliers"] == len(inl)
    assert np.linalg.norm(r["R"] - R) / np.linalg.norm(R) <= 1e-4
    assert np.linalg.norm(r["tvec"] - t) / np.linalg.norm(t) <= 1e-4


def test_batch_configure_restores_the_single_calibration(batch_units):
    units, P_l, P_r = batch_units
    c = _batch_context()
    c.batch_configure(BW, BH, B, P_l[0], P_r[0])
    keep = _submit(c, units, 0)
    before = _collect(c, 0, B)
    c.batch_calibrate(0, P_l, P_r)
    keep = _submit(c, units, 0)
    mixed = _collect(c, 0, B)
    assert not np.array_equal(mixed[1][0]["tvec"], before[1][0]["tvec"])
    c.batch_configure(BW, BH, B, P_l[0], P_r[0])
    keep = _submit(c, units, 0)
    after = _collect(c, 0, B)
    for i in range(B):
        _same_unit(after[i], before[i], f"unit {i}")
    c.close()


def test_refusals_leave_the_context_usable(ctx, small, batch_units, batch_alone):
    from visual_odom_b200 import capi
    units, P_l, P_r = batch_units
    c = _batch_context()
    c.batch_configure(BW, BH, B, P_l[0], P_r[0])

    def code(fn):
        with pytest.raises(capi.VoError) as e:
            fn()
        return e.value.code

    assert code(lambda: c.batch_calibrate(B - 1, P_l[:2], P_r[:2])) == capi.VO_E_INVALID       # past the last unit
    assert code(lambda: c.batch_calibrate(-1, P_l[:2], P_r[:2])) == capi.VO_E_INVALID
    assert c.lib.vo_batch_calibrate(c.h, 0, 0, P_l.ctypes.data, P_r.ctypes.data) == capi.VO_E_INVALID     # empty range
    assert c.lib.vo_batch_calibrate(c.h, 0, 1, None, P_r.ctypes.data) == capi.VO_E_INVALID
    assert c.lib.vo_batch_calibrate(c.h, 0, 1, P_l.ctypes.data, None) == capi.VO_E_INVALID
    keep = _submit(c, units, 0)
    assert code(lambda: c.batch_calibrate(0, P_l, P_r)) == capi.VO_E_INVALID                  # a submission in flight
    first = _collect(c, 0, B)
    for i in range(B):                                                                         # ran with calibration 0
        assert first[i][0]["n_valid"] > 0
    _same_unit(first[0], batch_alone[0], "unit 0 after the refusals")
    c.batch_calibrate(0, P_l, P_r)
    keep = _submit(c, units, 0)
    got = _collect(c, 0, B)
    for i in range(B):
        _same_unit(got[i], batch_alone[i], f"unit {i} after the refusals")
    c.close()
    # the multi-sequence entry point: NULL matrices, and the checks vo_mseq_begin_ex makes
    Pl, Pr, frames = small
    n = len(frames)
    lp, rp = (C.c_void_p * n)(), (C.c_void_p * n)()
    for q in range(n):
        lp[q], rp[q] = frames[q][0][0].ctypes.data, frames[q][0][1].ctypes.data
    Pl = np.ascontiguousarray(Pl, np.float32); Pr = np.ascontiguousarray(Pr, np.float32)
    w, h = SMALL[0], SMALL[1]
    assert ctx.lib.vo_mseq_begin_calib(ctx.h, n, w, h, None, Pr.ctypes.data, lp, rp, w, 1, 0) == capi.VO_E_INVALID
    assert ctx.lib.vo_mseq_begin_calib(ctx.h, n, w, h, Pl.ctypes.data, None, lp, rp, w, 1, 0) == capi.VO_E_INVALID
    assert ctx.lib.vo_mseq_begin_calib(ctx.h, 0, w, h, Pl.ctypes.data, Pr.ctypes.data, lp, rp, w, 1, 0) == capi.VO_E_INVALID
    assert ctx.lib.vo_mseq_begin_calib(ctx.h, n, w, h, Pl.ctypes.data, Pr.ctypes.data, lp, rp, w, 1, 4) == capi.VO_E_INVALID
    with pytest.raises(ValueError):
        ctx.mseq_begin([f[0][0] for f in frames], [f[0][1] for f in frames], Pl[:2], Pr[:2])
    # and the context goes on
    _check_against_alone(ctx, Pl, Pr, frames, _run_mseq(ctx, Pl, Pr, frames))
