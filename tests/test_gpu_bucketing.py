"""The sequence modes at any bucket grid, features per bucket, age gate and refill threshold, against the reference path.

vo_params.bucket_rows_divisor, features_per_bucket, bucket_age_threshold and refill_threshold replace the literals rows /
10, 1, 10 and 2000 of the reference's matchingFeatures() and Bucket::add_feature.  Every frame of vo_seq_* and vo_mseq_*
is held to the reference loop with the same values (test_oracle_bucketing.matching_features over oracle/ref_path.py's
cv2 backend): the record's counts, the four
point lists, the carried FeatureSet (points and ages) bit for bit, the inliers and [R|t] within POSE_TOL.  The entry paths
are run at eight features per bucket, where the live set passes 2000 points on every other frame and the refill is
skipped."""
import numpy as np
import pytest

from visual_odom_b200 import synth
from test_oracle_bucketing import matching_features

pytestmark = pytest.mark.gpu
POSE_TOL = 1e-8
CAP = 16384                    # max_features: the largest bound here is 1449 cells x 8 = 11592 points at divisor 20
NF = 9                         # frames per drive: eight pushes
DENSE = dict(features_per_bucket=8)
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")


def _drive(seed, w=1241, h=376, n=NF, r=synth.SEQ_STEP_R, t=synth.SEQ_STEP_T):
    base = synth.stereo_unit(w, h, seed)
    fr = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=np.asarray(r) * k, tvec=np.asarray(t) * k)
        fr.append((u["l1"], u["r1"]))
    return base["P_l"], base["P_r"], fr


_MOTION = {31: {}, 7: dict(r=(-0.002, 0.003, 0.0), t=(0.0, 0.0, -0.25)), 12: dict(t=(0.02, 0.0, -0.15))}


class _Drives(dict):
    """The three KITTI-sized drives, rendered on first use."""

    def __missing__(self, seed):
        self[seed] = _drive(seed, **_MOTION[seed])
        return self[seed]


DRIVES = _Drives()


def _context(**prm):
    from visual_odom_b200.capi import Context
    return Context(0, max_features=prm.pop("max_features", CAP), **prm)


def _oracle(P_l, P_r, frames, prm):
    """The reference main loop through ref_path (cv2) with the bucketing keywords: per frame the record's counts, the
    point lists, [R|t] (None below four valid points), the carried FeatureSet and whether the refill ran."""
    from oracle import ref_path
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    out = []
    for k in range(1, len(frames)):
        (l0, r0), (l1, r1) = frames[k - 1], frames[k]
        refilled = fs.size() < prm.get("refill_threshold", 2000)
        pL0, pR0, pL1, pR1, info = matching_features(l0, r0, l1, r1, fs, "cv2", **prm)
        rec = dict(n_features=len(info["bucketed"]), n_detected=len(ref_path.fast_cv2(l0)), n_tracked=len(info["kept_idx"]),
                   n_valid=len(pL0), l0=pL0, r0=pR0, l1=pL1, r1=pR1, R=None, refilled=refilled,
                   fs=(fs.points.copy(), fs.ages.copy()))
        if len(pL0) >= 4:
            X = ref_path.triangulate(P_l, P_r, pL0, pR0, "cv2")
            R, translation, inl, _ = ref_path.tracking_frame2frame(P_l, pL0, pL1, X, translation, "cv2")
            rec.update(R=R, t=translation.copy(), n_inliers=len(inl))
        out.append(rec)
    return out


def _check(got, state, ref, where):
    from visual_odom_b200.capi import VO_E_TOO_FEW_POINTS
    for key in ("n_features", "n_detected", "n_tracked", "n_valid"):
        assert got[key] == ref[key], f"{where}: {key} {got[key]} != {ref[key]}"
    for name in ("l0", "r0", "l1", "r1"):
        assert np.array_equal(got[name], ref[name]), f"{where}: {name}"
    pts, ages = state[0], state[1]
    assert np.array_equal(pts, ref["fs"][0]) and np.array_equal(ages, ref["fs"][1]), f"{where}: carried FeatureSet"
    if ref["R"] is None:
        assert got["pnp_status"] == VO_E_TOO_FEW_POINTS, where
        return
    assert got["n_inliers"] == ref["n_inliers"], f"{where}: inliers {got['n_inliers']} != {ref['n_inliers']}"
    d = max(np.abs(got["R"] - ref["R"]).max(), np.abs(got["tvec"] - ref["t"]).max())
    assert d <= POSE_TOL, (where, d)


def _push(c, P_l, P_r, frames, mono=False):
    """vo_seq_push over the drive: per frame (record, carried state)."""
    c.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    return [(c.seq_push(l, r, pts_cap=CAP, mono=mono), c.seq_state()) for l, r in frames[1:]]


def _same(a, b, where, mono=False):
    for key in INTS:
        assert a[key] == b[key], f"{where}: {key} {a[key]} != {b[key]}"
    for key in ("l0", "r0", "l1", "r1", "R", "tvec", "rvec") + (("ess_mask",) if mono else ()):
        assert np.array_equal(a[key], b[key]), f"{where}: {key}"


def _same_run(a, b, where):
    for k, ((ra, sa), (rb, sb)) in enumerate(zip(a, b), start=1):
        _same(ra, rb, f"{where} frame {k}")
        assert all(np.array_equal(x, y) for x, y in zip(sa, sb)), f"{where} frame {k}: carried state"


@pytest.fixture(scope="module")
def dense_alone(built):
    """Each drive alone through vo_seq_push at eight features per bucket, with its oracle."""
    c = _context(**DENSE)
    try:
        return {s: (_push(c, *DRIVES[s]), _oracle(*DRIVES[s], DENSE)) for s in _MOTION}
    finally:
        c.close()


# ----------------------------------------------------------------------------- the parameters against the oracle
GRIDS = [(k, d) for d in (10, 20) for k in (1, 2, 3, 8)] + [(1, 5), (1, 40)]


@pytest.mark.parametrize("k,divisor", GRIDS, ids=[f"k{k}-div{d}" for k, d in GRIDS])
def test_bucket_grid_and_density_match_the_reference(ctx, k, divisor):
    prm = dict(features_per_bucket=k, bucket_rows_divisor=divisor)
    P_l, P_r, frames = DRIVES[31]
    ref = _oracle(P_l, P_r, frames, prm)
    c = _context(**prm)
    try:
        got = _push(c, P_l, P_r, frames)
    finally:
        c.close()
    for i, ((g, st), r) in enumerate(zip(got, ref), start=1):
        _check(g, st, r, f"k={k} divisor={divisor} frame {i}")
    bs = 376 // divisor
    assert max(g["n_features"] for g, _ in got) <= (376 // bs + 1) * (1241 // bs + 1) * k
    if (k, divisor) == (1, 10):                     # the defaults: the same run as on a context without the fields
        _same_run(got, _push(ctx, P_l, P_r, frames), "default context")
    if (k, divisor) == (8, 10):
        assert not all(r["refilled"] for r in ref), "the live set never reached 2000 points"


@pytest.mark.parametrize("gate", (0, 1, 10, 1000))
def test_age_threshold_on_long_tracks(built, gate):
    """synth.blob_sequence keeps features alive for 10+ frames, so the gate decides which ones a cell admits."""
    P_l, P_r, frames = synth.blob_sequence()
    prm = dict(bucket_age_threshold=gate)
    ref = _oracle(P_l, P_r, frames, prm)
    c = _context(**prm)
    try:
        got = _push(c, P_l, P_r, frames)
    finally:
        c.close()
    for i, ((g, st), r) in enumerate(zip(got, ref), start=1):
        _check(g, st, r, f"gate={gate} frame {i}")
    if gate == 0:
        assert all(g["n_features"] == 0 for g, _ in got)
    if gate == 1000:                                # ages of 10 and more do enter here
        assert any((st[1][:len(st[0])] >= 10).any() for _, st in got)


@pytest.mark.parametrize("threshold", (0, 2000, 1000000))
def test_refill_threshold(built, threshold):
    prm = dict(DENSE, refill_threshold=threshold)
    P_l, P_r, frames = DRIVES[31]
    ref = _oracle(P_l, P_r, frames, prm)
    c = _context(**prm)
    try:
        got = _push(c, P_l, P_r, frames)
    finally:
        c.close()
    for i, ((g, st), r) in enumerate(zip(got, ref), start=1):
        _check(g, st, r, f"refill_threshold={threshold} frame {i}")
        assert g["n_detected"] > 10000, "n_detected counts the corners found whether or not they were appended"
    refills = [r["refilled"] for r in ref]
    if threshold == 0:
        assert not any(refills) and all(g["n_features"] == 0 for g, _ in got)
    elif threshold == 2000:
        assert refills[0] and not all(refills)
    else:
        assert all(refills)


# ----------------------------------------------------------------------------- every entry path at eight per bucket
def test_seq_push_and_submit_wait(built, dense_alone):
    P_l, P_r, frames = DRIVES[31]
    got, ref = dense_alone[31]
    for i, ((g, st), r) in enumerate(zip(got, ref), start=1):
        _check(g, st, r, f"vo_seq_push frame {i}")
    c = _context(**DENSE)
    try:
        c.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
        c.seq_submit(*frames[1])
        for k in range(1, len(frames)):
            if k + 1 < len(frames):
                c.seq_submit(*frames[k + 1])
            _same(c.seq_wait(pts_cap=CAP), got[k - 1][0], f"vo_seq_submit frame {k}")
        assert all(np.array_equal(x, y) for x, y in zip(c.seq_state(), got[-1][1]))
    finally:
        c.close()


def test_mseq_begin_three_sequences(built, dense_alone):
    seeds = (31, 7, 12)
    P_l = np.stack([DRIVES[s][0] for s in seeds]); P_r = np.stack([DRIVES[s][1] for s in seeds])
    c = _context(**DENSE)
    try:
        c.mseq_begin([DRIVES[s][2][0][0] for s in seeds], [DRIVES[s][2][0][1] for s in seeds], P_l, P_r)
        for k in range(1, NF):
            c.mseq_submit([DRIVES[s][2][k][0] for s in seeds], [DRIVES[s][2][k][1] for s in seeds])
            recs = c.mseq_wait(pts_cap=CAP)
            for q, s in enumerate(seeds):
                _same(recs[q], dense_alone[s][0][k - 1][0], f"sequence {q} frame {k}")
                _check(recs[q], c.mseq_state(q), dense_alone[s][1][k - 1], f"sequence {q} frame {k}")
    finally:
        c.close()


def test_mseq_begin_sized_two_kitti_sizes(built, dense_alone):
    other = _drive(9, 1226, 370)
    ref = _oracle(*other, DENSE)
    c = _context(**DENSE)
    try:
        alone = _push(c, *other)
        P_l = np.stack([DRIVES[31][0], other[0]]); P_r = np.stack([DRIVES[31][1], other[1]])
        fr = [DRIVES[31][2], other[2]]
        c.mseq_begin([f[0][0] for f in fr], [f[0][1] for f in fr], P_l, P_r)
        for k in range(1, NF):
            c.mseq_submit([f[k][0] for f in fr], [f[k][1] for f in fr])
            recs = c.mseq_wait(pts_cap=CAP)
            _same(recs[0], dense_alone[31][0][k - 1][0], f"1241 x 376 frame {k}")
            _same(recs[1], alone[k - 1][0], f"1226 x 370 frame {k}")
            _check(recs[1], c.mseq_state(1), ref[k - 1], f"1226 x 370 frame {k}")
    finally:
        c.close()


def test_mseq_open_and_start(built, dense_alone):
    from visual_odom_b200 import capi
    seeds = (31, 7)
    c = _context(**DENSE)
    try:
        c.mseq_open(2, 1241, 376)
        fr = [DRIVES[s][2] for s in seeds]
        c.mseq_submit([f[0][0] for f in fr], [f[0][1] for f in fr],
                      start={q: (DRIVES[s][0], DRIVES[s][1]) for q, s in enumerate(seeds)})
        assert all(r["status"] == capi.VO_MSEQ_STARTED for r in c.mseq_wait(pts_cap=CAP))
        for k in range(1, NF):
            c.mseq_submit([f[k][0] for f in fr], [f[k][1] for f in fr])
            recs = c.mseq_wait(pts_cap=CAP)
            for q, s in enumerate(seeds):
                _same(recs[q], dense_alone[s][0][k - 1][0], f"slot {q} frame {k}")
    finally:
        c.close()


def test_mseq_begin_device(built, dense_alone):
    torch = pytest.importorskip("torch")
    seeds = (31, 12)
    P_l = np.stack([DRIVES[s][0] for s in seeds]); P_r = np.stack([DRIVES[s][1] for s in seeds])
    dev = {s: [(torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda()) for l, r in DRIVES[s][2]] for s in seeds}
    torch.cuda.synchronize()
    c = _context(**DENSE)
    try:
        c.mseq_begin_device([dev[s][0][0] for s in seeds], [dev[s][0][1] for s in seeds], P_l, P_r)
        for k in range(1, NF):
            c.mseq_submit_device([dev[s][k][0] for s in seeds], [dev[s][k][1] for s in seeds])
            recs = c.mseq_wait(pts_cap=CAP)
            for q, s in enumerate(seeds):
                _same(recs[q], dense_alone[s][0][k - 1][0], f"sequence {q} frame {k}")
    finally:
        c.close()


def _mono_stage(c, P_l, rec, where):
    """The branch's record against vo_mono_rotation (the stage call held to cv2 by test_gpu_stages.py) on its lists."""
    from visual_odom_b200.capi import VoError
    focal = float(P_l[0, 0]); pp = (float(P_l[0, 2]), float(P_l[1, 2]))
    try:
        Rs, ms, its = c.mono_rotation(rec["l0"], rec["l1"], focal, pp)
    except VoError:
        assert rec["mono"]["status"] != 0 and np.array_equal(rec["R"], np.eye(3)), where
        return
    assert rec["mono"]["status"] == 0, where
    assert np.array_equal(rec["ess_mask"], ms) and np.array_equal(rec["R"], Rs), f"{where}: essential mask / rotation"
    assert rec["mono"]["ransac_iters"] == its, where


def test_mono_branch_in_both_modes(built, dense_alone):
    seeds = (31, 7)
    c = _context(**DENSE)
    try:
        c.set_option("mono_rotation", 1)
        got = _push(c, *DRIVES[31], mono=True)
        for k, ((g, st), (a, sa)) in enumerate(zip(got, dense_alone[31][0]), start=1):
            for key in ("n_features", "n_valid", "n_inliers", "pnp_status"):
                assert g[key] == a[key], (k, key)
            assert all(np.array_equal(x, y) for x, y in zip(st, sa)), k
            _check(dict(g, R=a["R"]), st, dense_alone[31][1][k - 1], f"vo_seq mono frame {k}")
            _mono_stage(c, DRIVES[31][0], g, f"vo_seq mono frame {k}")
        c.set_option("mono_rotation", 0)
        P_l = np.stack([DRIVES[s][0] for s in seeds]); P_r = np.stack([DRIVES[s][1] for s in seeds])
        c.mseq_begin([DRIVES[s][2][0][0] for s in seeds], [DRIVES[s][2][0][1] for s in seeds], P_l, P_r, mono_rotation=True)
        for k in range(1, NF):
            c.mseq_submit([DRIVES[s][2][k][0] for s in seeds], [DRIVES[s][2][k][1] for s in seeds])
            recs = c.mseq_wait(pts_cap=CAP, mono=True)
            _same(recs[0], got[k - 1][0], f"vo_mseq mono sequence 0 frame {k}", mono=True)
            _mono_stage(c, DRIVES[7][0], recs[1], f"vo_mseq mono sequence 1 frame {k}")
    finally:
        c.close()


def _launches_per_submission(c, frames, multi, mono):
    P_l, P_r, fr = frames
    if multi:
        c.mseq_begin([fr[0][0]] * 2, [fr[0][1]] * 2, P_l, P_r, mono_rotation=mono)
    else:
        c.set_option("mono_rotation", 1 if mono else 0)
        c.seq_begin(fr[0][0], fr[0][1], P_l, P_r)

    def step(k):
        if multi:
            c.mseq_submit([fr[k][0]] * 2, [fr[k][1]] * 2); c.mseq_wait(want_points=False, mono=mono)
        else:
            c.seq_submit(*fr[k]); c.seq_wait(want_points=False, mono=mono)
    for k in (1, 2):                          # the graphs of both buffer parities
        step(k)
    l0 = c.kernel_launches()
    for k in range(3, 6):
        step(k)
    c.set_option("mono_rotation", 0)
    return (c.kernel_launches() - l0) / 3


def test_launches_per_submission_do_not_depend_on_the_density(built):
    for prm in (dict(), DENSE, dict(features_per_bucket=3, bucket_rows_divisor=20)):
        c = _context(**prm)
        try:
            for multi in (False, True):
                assert _launches_per_submission(c, DRIVES[31], multi, False) == 30, (prm, multi)
                assert _launches_per_submission(c, DRIVES[31], multi, True) == 49, (prm, multi)
        finally:
            c.close()


# ----------------------------------------------------------------------------- refusals and the capacity rule
def test_refusals_leave_the_context_usable(built, dense_alone):
    from visual_odom_b200 import capi
    P_l, P_r, frames = DRIVES[31]
    l, r = frames[0]
    for field, value in (("features_per_bucket", 0), ("bucket_rows_divisor", -1)):
        with pytest.raises(capi.VoError) as e:
            _context(**{field: value})
        assert e.value.code == capi.VO_E_INVALID, field
    # rows / divisor == 0: 376 / 400
    c = _context(bucket_rows_divisor=400)
    try:
        for call in (lambda: c.seq_begin(l, r, P_l, P_r), lambda: c.mseq_begin([l, l], [r, r], P_l, P_r),
                     lambda: c.mseq_open(2, 1241, 376)):
            with pytest.raises(capi.VoError) as e:
                call()
            assert e.value.code == capi.VO_E_UNSUPPORTED and "rows/400" in str(e.value), str(e.value)
    finally:
        c.close()
    # 2992 points at eight per bucket against 2048: begin, begin, open; then a start above 3000 in a run that fits
    c = _context(features_per_bucket=8, max_features=2048)
    try:
        for call in (lambda: c.seq_begin(l, r, P_l, P_r), lambda: c.mseq_begin([l, l], [r, r], P_l, P_r),
                     lambda: c.mseq_open(2, 1241, 376)):
            with pytest.raises(capi.VoError) as e:
                call()
            assert e.value.code == capi.VO_E_CAPACITY and "2992" in str(e.value) and "2048" in str(e.value), str(e.value)
    finally:
        c.close()
    c = _context(features_per_bucket=8, max_features=3000)
    try:
        small = _drive(31, 1241, 200, n=2)
        c.mseq_open(2, 1241, 376)
        with pytest.raises(capi.VoError) as e:       # 1241 x 200: 11 x 63 cells x 8 = 5544 points
            c.mseq_submit([small[2][0][0], None], [small[2][0][1], None], start={0: (small[0], small[1])})
        assert e.value.code == capi.VO_E_CAPACITY and "5544" in str(e.value), str(e.value)
        c.mseq_submit([frames[0][0], None], [frames[0][1], None], start={0: (P_l, P_r)})
        c.mseq_wait()
        for k in range(1, NF):
            c.mseq_submit([frames[k][0], None], [frames[k][1], None])
            _same(c.mseq_wait(pts_cap=CAP)[0], dense_alone[31][0][k - 1][0], f"after the refusals, frame {k}")
        _same_run(_push(c, P_l, P_r, frames), dense_alone[31][0], "vo_seq after the refusals")
    finally:
        c.close()


def test_scratch_and_graphs_follow_the_bound(built, dense_alone):
    """k = 8 on one context: a vo_seq_* run (2992-point bound), a vo_mseq_begin_sized run with a larger grid (1241 x 200:
    5544), then the first run again, each with the mono branch (whose scratch grows with the bound): each equals the same
    run on a fresh context."""
    tall = DRIVES[31]
    wide = _drive(5, 1241, 200)

    def seq(c):
        c.set_option("mono_rotation", 1)
        out = _push(c, *tall, mono=True)
        c.set_option("mono_rotation", 0)
        return out

    def mseq(c):
        P_l = np.stack([tall[0], wide[0]]); P_r = np.stack([tall[1], wide[1]])
        fr = [tall[2], wide[2]]
        c.mseq_begin([f[0][0] for f in fr], [f[0][1] for f in fr], P_l, P_r, mono_rotation=True)
        out = []
        for k in range(1, NF):
            c.mseq_submit([f[k][0] for f in fr], [f[k][1] for f in fr])
            out.append(c.mseq_wait(pts_cap=CAP, mono=True))
        return out

    def fresh(run):
        f = _context(**DENSE)
        try:
            return run(f)
        finally:
            f.close()

    c = _context(**DENSE)
    try:
        first, sized, again = seq(c), mseq(c), seq(c)
    finally:
        c.close()
    want_seq, want_sized = fresh(seq), fresh(mseq)
    for k in range(NF - 1):
        for got in (first, again):
            _same(got[k][0], want_seq[k][0], f"vo_seq frame {k + 1}", mono=True)
            assert all(np.array_equal(x, y) for x, y in zip(got[k][1], want_seq[k][1]))
        for q in range(2):
            _same(sized[k][q], want_sized[k][q], f"vo_mseq_begin_sized sequence {q} frame {k + 1}", mono=True)
    assert max(r[1]["n_features"] for r in sized) > 2992 and max(g["n_features"] for g, _ in first) <= 2992
