"""The run-time LK, validity-filter and PnP parameters of vo_params away from the reference's literals, through the C-ABI:
every result bit for bit as cv2 (and the oracle, pinned to cv2 at the same values in test_oracle_params.py) gives it.

- vo_lk_track and vo_circular_match at every pyramid depth the library accepts (up to 8 images: 32 phases per feature in
  the ring), at iteration counts inside and outside calcOpticalFlowPyrLK's clamp, at minEig thresholds including ones a
  quarter ulp from a window's minEig, and on flat and saturated windows at threshold 0 (the D < FLT_EPSILON rejection);
  the 8-image pyramid and the logged thresholds under every LK launch configuration (work items of 1 to 16 phases and
  the whole ring).
- vo_pnp_ransac at iteration counts on and around the wave boundaries of the PnP launch (32, 128) and at or below 0.
- circ_threshold through vo_frame_batch and the sequence mode.
- one context with every one of these parameters off its default through vo_frame_batch, vo_seq_push, vo_seq_submit and
  vo_mseq_*: each against the reference's glue at the same values, and the modes against each other.
- a shallower pyramid lets vo_mseq_begin_sized take sizes that the default depth separates."""
import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")
import test_oracle_params as OP  # noqa: E402

POSE_TOL = 1e-8
SPANS = (0, 1, 2, 3, 5, 7, 16, 32)           # 0 = automatic; 32 = the whole ring of an 8-image pyramid in one item
CONFIGS = [dict(lk_span=s) for s in SPANS]
CONFIG_IDS = ["-".join(f"{k}={v}" for k, v in c.items()) for c in CONFIGS]


def _context(opts=None, **params):
    from visual_odom_b200.capi import Context
    c = Context(0, max_features=8192, **params)
    for k, v in (opts or {}).items():
        c.set_option(k, v)
    return c


def _lk_params(kw):
    names = dict(max_level="lk_max_level", max_iters="lk_max_iters", epsilon="lk_epsilon", min_eig="lk_min_eig")
    return {names[k]: v for k, v in kw.items()}


def _check_track(c, prev, nxt, pts, kw, where):
    ref, orc = OP.lk_both(prev, nxt, pts, **kw)
    got = c.lk_track(prev, nxt, pts)
    OP.assert_lk_equal(ref, got, f"{where}: GPU vs cv2")
    OP.assert_lk_equal(orc[:3], got, f"{where}: GPU vs oracle")
    return ref


def _ring_images(prev, nxt):
    """(l0, r0, l1, r1) so that every call of the ring L0->R0->R1->L1->L0 tracks between the two views."""
    return prev, nxt, nxt, prev


def _check_ring(c, imgs, pts, kw, where):
    from oracle import ref_path
    fs = ref_path.FeatureSet()
    fs.points = pts.copy(); fs.ages = np.arange(len(pts), dtype=np.int32) % 5
    ages0 = fs.ages.copy()
    ref = ref_path.circular_matching(*imgs, pts, fs, backend="cv2", **kw)
    got = c.circular_match(*imgs, pts, ages=ages0)
    assert np.array_equal(got["status4"], ref["raw"]["status"]), f"{where}: ring status"
    for k, name in enumerate(("r0", "r1", "l1", "l0_ret")):
        bad = np.nonzero((got["raw4"][k] != ref["raw"][name]).any(1))[0]
        assert len(bad) == 0, f"{where}: raw {name} differs at {len(bad)} points, first {bad[:8]}"
    assert np.array_equal(got["kept_idx"], ref["kept_idx"]), where
    for name in ("l0", "r0", "l1", "r1", "l0_ret"):
        assert np.array_equal(got[name], ref[name]), f"{where}: {name}"
    assert np.array_equal(got["ages"], fs.ages), where
    return ref


# ----------------------------------------------------------------------------- LK grid (default launch configuration)
LK_CASES = ([("level", name, dict(max_level=m)) for name in OP.LK_IMAGES for m in range(8)]
            + [("iters", "small", dict(max_iters=i, epsilon=0.0)) for i in OP.LK_ITERS]
            + [("min_eig", name, dict(min_eig=t)) for name in ("small", "kitti") for t in OP.LK_MIN_EIGS])


@pytest.mark.parametrize("case", LK_CASES, ids=[f"{k}-{n}-{'-'.join(f'{a}={b}' for a, b in kw.items())}" for k, n, kw in LK_CASES])
def test_lk_track_and_ring_parameters(built, case):
    _, name, kw = case
    prev, nxt, pts = OP.lk_image(name)
    c = _context(**_lk_params(kw))
    try:
        ref = _check_track(c, prev, nxt, pts, kw, f"{name} {kw}")
        assert 0 < ref[1].sum() < len(pts)
        _check_ring(c, _ring_images(prev, nxt), pts, kw, f"{name} {kw} ring")
    finally:
        c.close()


def test_flat_and_saturated_windows_at_threshold_zero(built):
    prev, nxt, pts = OP.flat_pair()
    kw = dict(min_eig=0.0)
    c = _context(lk_min_eig=0.0)
    try:
        ref = _check_track(c, prev, nxt, pts, kw, "flat blocks")
        assert (ref[1][:108] == 0).sum() >= 12
        _check_ring(c, _ring_images(prev, nxt), pts, kw, "flat blocks ring")
    finally:
        c.close()


# ----------------------------------------------------------------------------- every launch configuration
@pytest.fixture(scope="module")
def thresholds():
    """16 thresholds from the small pair's event log (8 a quarter ulp above a level-0 minEig, 8 below)."""
    picked = OP.logged_thresholds()[::25]
    return [t for _, a, b in picked for t in (a, b)]


@pytest.mark.parametrize("i", range(len(CONFIGS)), ids=CONFIG_IDS)
def test_eight_level_pyramid_under_every_launch_configuration(built, i):
    """2816 x 2816 at lk_max_level 7: 8 images, 8 phases per call, 32 per ring; the level geometry and TMA descriptors of
    levels 4 to 7 are read."""
    prev, nxt, pts = OP.lk_image("deep")
    kw = dict(max_level=7)
    c = _context(CONFIGS[i], lk_max_level=7)
    try:
        _check_track(c, prev, nxt, pts, kw, f"deep {CONFIG_IDS[i]}")
        _check_ring(c, _ring_images(prev, nxt), pts, kw, f"deep ring {CONFIG_IDS[i]}")
    finally:
        c.close()


@pytest.mark.parametrize("i", range(len(CONFIGS)), ids=CONFIG_IDS)
def test_logged_min_eig_thresholds_under_every_launch_configuration(built, thresholds, i):
    """A threshold that rounds to a window's minEig keeps that window, as cv2's float comparison does; every start is
    tracked at each threshold."""
    prev, nxt, pts = OP.lk_image("small")
    for t in thresholds:
        c = _context(CONFIGS[i], lk_min_eig=t)
        try:
            _check_track(c, prev, nxt, pts, dict(min_eig=t), f"threshold {t!r} {CONFIG_IDS[i]}")
        finally:
            c.close()


def test_logged_min_eig_thresholds_one_start_each(built):
    """All 400 logged thresholds (200 windows, both sides), each with its own start, on the default configuration."""
    prev, nxt, _ = OP.lk_image("small")
    kept = 0
    for p, t_above, t_below in OP.logged_thresholds():
        for t in (t_above, t_below):
            c = _context(lk_min_eig=t)
            try:
                ref = _check_track(c, prev, nxt, p.reshape(1, 2), dict(min_eig=t), f"start {p} threshold {t!r}")
                kept += int(ref[1][0])
            finally:
                c.close()
    assert kept >= 300


# ----------------------------------------------------------------------------- PnP
GPU_PNP_ITERS = (-5, 0, 1, 2, 31, 32, 33, 127, 128, 129, 500, 2000)
GPU_PNP_SETS = {"s300": (300, 0.1, 0.2, 4), "s300b": (300, 0.05, 0.3, 5)}


@pytest.fixture(scope="module")
def pnp_sets():
    return {k: synth.pnp_stress_set(*v[:3], seed=v[3])[:3] for k, v in GPU_PNP_SETS.items()}


@pytest.mark.parametrize("iterations", GPU_PNP_ITERS)
def test_pnp_ransac_iterations_around_the_wave_boundaries(built, pnp_sets, iterations):
    """Inlier lists as cv2's, RANSAC iterations as the oracle's and [R|t] within 1e-8 of cv2, at reprojection errors
    0.1 and 2.0 and confidences 0.5 and 0.99.  On the 300-point set at 0.1 px and 0.99 RANSAC runs to the cap, so the
    waves [0, 32), [32, 128), [128, its) end where the count says; a count <= 0 runs one iteration, as cv2 does."""
    from oracle import pnp_ref
    capped = no_model = 0
    for name, (X, x, K) in pnp_sets.items():
        for reproj in (0.1, 2.0):
            for conf in (0.5, 0.99):
                where = f"{name} iterations={iterations} reproj={reproj} confidence={conf}"
                ok, rv, tv, inl = OP.cv2_pnp(X, x, K, iterations, reproj, conf)
                orc = pnp_ref.solve_pnp_ransac(X, x, K, np.zeros(3), OP.T_PREV, iterations=iterations, reproj=reproj,
                                               confidence=conf)
                assert ok == orc["ok"] and np.array_equal(orc["inliers"], inl), where
                c = _context(pnp_iterations=iterations, pnp_reproj_error=reproj, pnp_confidence=conf)
                try:
                    got = c.pnp_ransac(X, x, K, tvec0=OP.T_PREV)
                finally:
                    c.close()
                assert np.array_equal(got["inliers"], inl), f"{where}: {len(got['inliers'])} inliers, cv2 {len(inl)}"
                assert got["iters"] == orc["iters"], f"{where}: {got['iters']} RANSAC iterations, oracle {orc['iters']}"
                capped += orc["iters"] == max(iterations, 1)
                if not ok:                  # no model with more than 4 inliers (VO_PNP_NO_MODEL): the caller's guess
                    no_model += 1
                    assert np.array_equal(got["R"], np.eye(3)) and np.array_equal(got["tvec"], OP.T_PREV), where
                    continue
                d = max(np.abs(got["rvec"] - rv).max(), np.abs(got["tvec"] - tv).max(), np.abs(got["R"] - cv2.Rodrigues(rv)[0]).max())
                assert d <= POSE_TOL, (where, d)
    assert capped >= 1
    if iterations <= 2:                 # the 300-point set finds a model in its first subset, the other one does not
        assert 0 < no_model < 8


# ----------------------------------------------------------------------------- drives through the whole path
NF = 5


def _drive(w, h, seed, r=synth.SEQ_STEP_R, t=synth.SEQ_STEP_T):
    base = synth.stereo_unit(w, h, seed)
    fr = [(base["l0"], base["r0"])]
    for k in range(1, NF):
        u = synth.stereo_unit(w, h, seed, rvec=np.asarray(r) * k, tvec=np.asarray(t) * k)
        fr.append((u["l1"], u["r1"]))
    return base["P_l"], base["P_r"], fr


def _glue(prm):
    """ref_path keywords of a vo_params dict."""
    lk = dict(max_level=prm.get("lk_max_level", 3), max_iters=prm.get("lk_max_iters", 30), epsilon=prm.get("lk_epsilon", 0.01),
              min_eig=prm.get("lk_min_eig", 1e-3))
    pnp = dict(iterations=prm.get("pnp_iterations", 500), reproj=float(np.float32(prm.get("pnp_reproj_error", 0.5))),
               confidence=prm.get("pnp_confidence", float(np.float32(0.999))))
    return lk, prm.get("circ_threshold", 0), pnp


def _glue_drive(P_l, P_r, frames, prm):
    """The reference's main loop through ref_path (cv2) at the parameters: per frame the record's counts, point lists,
    [R|t] (None where cv2 would throw: fewer than four valid points) and frame_pose."""
    from oracle import ref_path
    lk, circ, pnp = _glue(prm)
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    out = []
    for k in range(1, len(frames)):
        (l0, r0), (l1, r1) = frames[k - 1], frames[k]
        pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, "cv2", circ_threshold=circ, **lk)
        rec = dict(n_features=len(info["bucketed"]), n_tracked=len(info["kept_idx"]), n_valid=len(pL0),
                   l0=pL0, r0=pR0, l1=pL1, r1=pR1, bucketed=info["bucketed"].copy(), R=None)
        if len(pL0) >= 4:
            X = ref_path.triangulate(P_l, P_r, pL0, pR0, "cv2")
            R, translation, inl, _ = ref_path.tracking_frame2frame(P_l, pL0, pL1, X, translation, "cv2", **pnp)
            frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
            rec.update(R=R, t=translation.copy(), n_inliers=len(inl))
        rec["pose"] = frame_pose.copy()
        out.append(rec)
    return out


def _check_glue(got, ref, where, pose=None):
    for key in ("n_features", "n_tracked", "n_valid"):
        assert got[key] == ref[key], f"{where}: {key} {got[key]} != {ref[key]}"
    for name in ("l0", "r0", "l1", "r1"):
        assert np.array_equal(got[name], ref[name]), f"{where}: {name}"
    if ref["R"] is None:
        from visual_odom_b200.capi import VO_E_TOO_FEW_POINTS
        assert got["pnp_status"] == VO_E_TOO_FEW_POINTS, where
        return
    assert got["n_inliers"] == ref["n_inliers"], f"{where}: inliers {got['n_inliers']} != {ref['n_inliers']}"
    d = max(np.abs(got["R"] - ref["R"]).max(), np.abs(got["tvec"] - ref["t"]).max())
    assert d <= POSE_TOL, (where, d)
    if pose is not None:
        assert np.abs(pose - ref["pose"]).max() <= 1e-6 * max(1.0, np.abs(ref["pose"]).max()), f"{where}: frame_pose"


def _seq_push_run(c, P_l, P_r, frames):
    c.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    out = []
    for k in range(1, len(frames)):
        out.append(c.seq_push(*frames[k]))
        out[-1]["pose"] = c.seq_pose()
    return out


def _seq_submit_run(c, P_l, P_r, frames):
    c.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    c.seq_submit(*frames[1])
    out = []
    for k in range(1, len(frames)):
        if k + 1 < len(frames):
            c.seq_submit(*frames[k + 1])
        out.append(c.seq_wait())
    return out


def _same(a, b, where, ints=("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")):
    for key in ints:
        assert a[key] == b[key], f"{where}: {key} {a[key]} != {b[key]}"
    for key in ("l0", "r0", "l1", "r1", "R", "tvec", "rvec"):
        assert np.array_equal(a[key], b[key]), f"{where}: {key}"


# a batched unit handed its points neither detects nor buckets: its records agree with the sequence's from the ring on
BATCH_INTS = ("n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")


def _batch_units(c, P_l, P_r, frames, seq, prm):
    """vo_frame_batch with one unit per frame of the drive: the points the sequence bucketed and the sequence's previous
    translation as the guess; records and point lists."""
    from visual_odom_b200.capi import VO_OK
    w, h = frames[0][0].shape[1], frames[0][0].shape[0]
    units = []
    for k in range(1, len(frames)):
        t_prev = tuple(seq[k - 2]["tvec"]) if k >= 2 and seq[k - 2]["pnp_status"] == VO_OK else (0.0, 0.0, 0.0)
        (l0, r0), (l1, r1) = frames[k - 1], frames[k]
        units.append(dict(l0=l0, r0=r0, l1=l1, r1=r1, pts=seq[k - 1]["bucketed"], t_prev=t_prev))
    c.batch_configure(w, h, len(units), P_l, P_r)
    arr, keep, pitch = c.make_units(units)
    res = c.frame_batch(arr, pitch)
    for i, r in enumerate(res):
        r.update({k: v for k, v in c.batch_fetch(i, r).items() if k in ("l0", "r0", "l1", "r1")})
    return res


@pytest.mark.parametrize("circ", OP.CIRC_THRESHOLDS)
def test_circ_threshold_through_the_batched_and_sequence_modes(built, circ):
    P_l, P_r, frames = _drive(1241, 376, 31)
    prm = dict(circ_threshold=circ)
    ref = _glue_drive(P_l, P_r, frames, prm)
    c = _context(**prm)
    try:
        seq = _seq_push_run(c, P_l, P_r, frames)
        for k, (g, r) in enumerate(zip(seq, ref), start=1):
            _check_glue(g, r, f"circ={circ} vo_seq_push frame {k}", pose=g["pose"])
        for k, (g, r) in enumerate(zip(_batch_units(c, P_l, P_r, frames, [dict(s, bucketed=r["bucketed"]) for s, r in zip(seq, ref)], prm),
                                       seq), start=1):
            _same(g, r, f"circ={circ} vo_frame_batch unit {k} vs vo_seq_push", ints=BATCH_INTS)
    finally:
        c.close()
    if circ < 0:
        assert all(r["n_valid"] == 0 for r in ref)
    else:
        assert all(r["n_valid"] > 50 for r in ref)


OFF_DEFAULTS = dict(lk_max_level=4, lk_max_iters=12, lk_epsilon=0.02, lk_min_eig=4e-3, circ_threshold=1, pnp_iterations=100,
                    pnp_reproj_error=1.0, pnp_confidence=0.99)


def test_every_parameter_off_its_default_in_every_mode(built):
    """One context at OFF_DEFAULTS (1241 x 376 at lk_max_level 4: 5 pyramid images): vo_seq_push against the glue, and
    vo_seq_submit / vo_seq_wait, vo_frame_batch and vo_mseq_* with two sequences against vo_seq_push, bit for bit."""
    P_l, P_r, frames = _drive(1241, 376, 7)
    _, _, frames2 = _drive(1241, 376, 12, r=(-0.002, 0.003, 0.0), t=(0.0, 0.0, -0.25))
    from oracle import cref
    assert cref.Pyramid(frames[0][0], max_level=4).nlevels() == 5
    refs = [_glue_drive(P_l, P_r, fr, OFF_DEFAULTS) for fr in (frames, frames2)]
    c = _context(**OFF_DEFAULTS)
    try:
        seqs = [_seq_push_run(c, P_l, P_r, fr) for fr in (frames, frames2)]
        for q in range(2):
            for k, (g, r) in enumerate(zip(seqs[q], refs[q]), start=1):
                _check_glue(g, r, f"drive {q} vo_seq_push frame {k}", pose=g["pose"])
                assert r["n_valid"] > 50 and r["n_inliers"] > 20
        for k, (g, r) in enumerate(zip(_seq_submit_run(c, P_l, P_r, frames), seqs[0]), start=1):
            _same(g, r, f"vo_seq_submit frame {k}")
        batch = _batch_units(c, P_l, P_r, frames, [dict(s, bucketed=r["bucketed"]) for s, r in zip(seqs[0], refs[0])], OFF_DEFAULTS)
        for k, (g, r) in enumerate(zip(batch, seqs[0]), start=1):
            _same(g, r, f"vo_frame_batch unit {k}", ints=BATCH_INTS)
        c.mseq_begin([frames[0][0], frames2[0][0]], [frames[0][1], frames2[0][1]], np.stack([P_l, P_l]), np.stack([P_r, P_r]))
        for k in range(1, NF):
            c.mseq_submit([frames[k][0], frames2[k][0]], [frames[k][1], frames2[k][1]])
            recs = c.mseq_wait()
            for q in range(2):
                _same(recs[q], seqs[q][k - 1], f"vo_mseq sequence {q} frame {k}")
                assert np.array_equal(c.mseq_pose(q), seqs[q][k - 1]["pose"])
    finally:
        c.close()


def test_a_shallower_pyramid_lets_mseq_begin_sized_take_two_depths_of_the_default(built):
    """120 x 233 has 3 pyramid images at lk_max_level 3 and 640 x 240 has 4, so the default refuses the pair in one run; at
    lk_max_level 1 both have 2, and each sequence is bit for bit its run alone."""
    from visual_odom_b200.capi import VO_E_UNSUPPORTED, VoError
    drives = [_drive(640, 240, 31), _drive(120, 233, 8, r=(0.0, 0.002, 0.0), t=(0.0, 0.0, -0.15))]
    lefts = [d[2][0][0] for d in drives]; rights = [d[2][0][1] for d in drives]
    P_l = np.stack([d[0] for d in drives]); P_r = np.stack([d[1] for d in drives])
    d = _context()
    try:
        with pytest.raises(VoError) as e:
            d.mseq_begin(lefts, rights, P_l, P_r)
        assert e.value.code == VO_E_UNSUPPORTED and "pyramid levels" in str(e.value)
    finally:
        d.close()
    c = _context(lk_max_level=1)
    try:
        alone = [_seq_push_run(c, P_l[q], P_r[q], drives[q][2]) for q in range(2)]
        c.mseq_begin(lefts, rights, P_l, P_r)
        for k in range(1, NF):
            c.mseq_submit([dr[2][k][0] for dr in drives], [dr[2][k][1] for dr in drives])
            recs = c.mseq_wait()
            for q in range(2):
                _same(recs[q], alone[q][k - 1], f"sequence {q} frame {k}")
                assert np.array_equal(c.mseq_pose(q), alone[q][k - 1]["pose"])
    finally:
        c.close()
    assert all(a[-1]["n_valid"] > 10 for a in alone)
