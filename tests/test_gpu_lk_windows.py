"""LK windows other than the reference's 21x21 (vo_params.lk_win from 3 to 32, k_lk_win in csrc/lk_win.cu), bit for bit
against the oracle (oracle/lk_ref.c, pinned to cv2 at every window by test_oracle_lk_windows.py) and cv2:

- vo_create accepts 3..32 and refuses the rest; a slot's or a unit's window other than the context's is still refused;
- vo_lk_track and vo_circular_match at every window on the scenes of lk_window_scenes.py, and the window-dependent pyramid
  depth of a 100 x 44 image; saturated blocks at 32 x 32;
- the minEig and epsilon decisions at their edges at W = 7 and 32, from thresholds read off the oracle's event log;
- at W = 5, 15 and 31: vo_frame_batch and vo_batch_submit / vo_batch_wait with graphs on and off and the SM partition at 0
  and 8 SMs, the sequence mode over 12 frames against the reference's glue, vo_mseq_begin_sized with two sizes against
  each sequence run alone, and frames already in GPU memory against the same frames from the host."""
import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")
import lk_window_scenes as S  # noqa: E402
from test_gpu_params import _same  # noqa: E402
from test_gpu_path import check_unit  # noqa: E402

POSE_TOL = 1e-8
MODE_WINDOWS = (5, 15, 31)


def _context(win, opts=None, **params):
    from visual_odom_b200.capi import Context
    c = Context(0, lk_win=win, **dict(dict(max_features=2048), **params))
    for k, v in (opts or {}).items():
        c.set_option(k, v)
    return c


@pytest.fixture(scope="module")
def scenes(built):
    return {name: make() for name, make in S.SCENES.items()}


@pytest.fixture(scope="module")
def ring_unit(built):
    from oracle import cref
    u = synth.stereo_unit(1241, 376, 5)
    corners, _ = cref.fast_detect(u["l0"])
    rng = np.random.default_rng(5)
    out = np.stack([rng.uniform(-40, 1281, 60), rng.uniform(-40, 416, 60)], 1).astype(np.float32)
    return u, np.concatenate([synth.select_features(corners, 1200), out])


def _assert_track(got, ref, what):
    go, gs, ge = got
    ro, rs, re = ref
    assert np.array_equal(gs, rs), f"{what}: status differs at {np.nonzero(gs != rs)[0][:8]}"
    bad = np.nonzero((go != ro).any(1))[0]
    assert len(bad) == 0, f"{what}: positions differ at {len(bad)} points, first {bad[:8]}"
    assert np.array_equal(ge[rs == 1], re[rs == 1]), f"{what}: err"


def _check_track(c, a, b, pts, win, what, **kw):
    ref = S.lk(a, b, pts, win, "c", **kw)
    cvr = S.lk(a, b, pts, win, "cv2", **kw)
    got = c.lk_track(a, b, pts)
    _assert_track(got, ref, f"{what} vs oracle")
    _assert_track(got, cvr, f"{what} vs cv2")
    return ref


def _check_ring(c, imgs, pts, win, what):
    from oracle import ref_path
    got = None
    for backend in ("c", "cv2"):
        fs = ref_path.FeatureSet()
        fs.points = pts.copy(); fs.ages = np.arange(len(pts), dtype=np.int32) % 5
        if got is None:
            got = c.circular_match(*imgs, pts, ages=fs.ages.copy())
        ref = S.circular_matching(*imgs, pts, fs, win, backend)
        where = f"{what} vs {backend}"
        assert np.array_equal(got["status4"], ref["raw"]["status"]), f"{where}: ring status"
        for k, name in enumerate(("r0", "r1", "l1", "l0_ret")):
            bad = np.nonzero((got["raw4"][k] != ref["raw"][name]).any(1))[0]
            assert len(bad) == 0, f"{where}: raw {name} differs at {len(bad)} points, first {bad[:8]}"
        assert np.array_equal(got["kept_idx"], ref["kept_idx"]), where
        for name in ("l0", "r0", "l1", "r1", "l0_ret"):
            assert np.array_equal(got[name], ref[name]), f"{where}: {name}"
        assert np.array_equal(got["ages"], fs.ages), where
    return got


# ----------------------------------------------------------------------------- the parameter
def test_create_accepts_3_to_32_and_refuses_the_rest(built):
    from visual_odom_b200 import capi
    for win in S.WINDOWS:
        _context(win, max_features=64).close()
    for win, rc, msg in ((1, capi.VO_E_INVALID, "lk_win=1"), (2, capi.VO_E_INVALID, "lk_win=2"),
                         (0, capi.VO_E_INVALID, "lk_win=0"), (33, capi.VO_E_UNSUPPORTED, "from 3 to 32")):
        with pytest.raises(capi.VoError) as e:
            _context(win)
        assert e.value.code == rc and msg in str(e.value), (win, str(e.value))
    u = synth.stereo_unit(640, 240, 1)
    c = _context(15)
    try:
        for other in (21, 14):
            with pytest.raises(capi.VoError) as e:
                c.mseq_params(0, [None, dict(lk_win=other)])
            assert e.value.code == capi.VO_E_UNSUPPORTED and "context-wide" in str(e.value) and "slot 1" in str(e.value)
        c.batch_configure(640, 240, 2, u["P_l"], u["P_r"])
        with pytest.raises(capi.VoError) as e:
            c.batch_params(0, [dict(lk_win=21)])
        assert e.value.code == capi.VO_E_UNSUPPORTED and "context-wide" in str(e.value)
        c.mseq_params(0, [dict(lk_win=15)])                 # the context's own window is accepted
    finally:
        c.close()


# ----------------------------------------------------------------------------- every window
@pytest.mark.parametrize("win", S.WINDOWS)
def test_lk_track_and_circular_match_at_every_window(scenes, ring_unit, win):
    from oracle import cref
    c = _context(win)
    try:
        for name, (a, b, pts) in scenes.items():
            ref = _check_track(c, a, b, pts, win, f"{name} W={win}")
            assert 0 < ref[1].sum() < len(pts)
        u, pts = ring_unit
        got = _check_ring(c, (u["l0"], u["r0"], u["l1"], u["r1"]), pts, win, f"stereo ring W={win}")
        assert len(got["kept_idx"]) > 0
        a, b, pts = scenes["noise"]
        _check_ring(c, (a, b, b, a), pts, win, f"noise ring W={win}")
        # the pyramid depth follows the window: 100 x 44 has 4 images at W <= 10 ... 1 at W >= 22
        small = synth.stereo_unit(100, 44, 9, scene="v0")
        assert cref.Pyramid(small["l0"], win).nlevels() == (4 if win <= 5 else 3 if win <= 10 else 2 if win <= 21 else 1)
        spts = np.array([[20.5, 12.25], [50, 22], [80.75, 30.5], [5, 40], [99, 43], [-3, 10], [102, 20]], np.float32)
        _check_track(c, small["l0"], small["r0"], spts, win, f"100x44 W={win}")
    finally:
        c.close()


def test_saturated_blocks_at_the_largest_window(built):
    """0 / 255 blocks at KITTI size with a 32 x 32 window: the b sums reach about 3e9, past int32; the float chains that
    cv2 adds are formed from pair sums that stay far below it."""
    a, b, pts = S.block_pair(1241, 376, seed=9, n=2000)
    c = _context(32)
    try:
        ref = _check_track(c, a, b, pts, 32, "saturated W=32")
        assert ref[1].sum() > len(pts) // 2
        _check_ring(c, (a, b, b, a), pts, 32, "saturated ring W=32")
    finally:
        c.close()


# ----------------------------------------------------------------------------- decision edges
def _log(a, b, pts, win, **kw):
    from oracle import cref
    return cref.lk_track(a, b, pts, win=win, return_log=True, **kw)[-1]


@pytest.mark.parametrize("win", (7, 32))
def test_min_eig_threshold_at_a_logged_min_eig(scenes, win):
    """lk_min_eig equal to a start's level-0 minEig keeps the window (minEig < threshold rejects); the next float up
    rejects it."""
    from oracle import cref
    a, b, pts = scenes["noise"]
    log = _log(a, b, pts, win)
    ev = log[(log["kind"] == cref.EV_SETUP) & (log["level"] == 0)][0]
    p = pts[ev["pt"]:ev["pt"] + 1]
    m = np.float32(ev["min_eig"])
    for t, kind in ((m, cref.EV_SETUP), (np.nextafter(m, np.float32(np.inf)), cref.EV_REJECT)):
        lg = _log(a, b, p, win, min_eig=float(t))
        assert lg[(lg["level"] == 0) & (lg["iter"] == -1)]["kind"][0] == kind, (win, t)
        c = _context(win, lk_min_eig=float(t))
        try:
            ref = _check_track(c, a, b, p, win, f"W={win} min_eig={float(t)!r}", min_eig=float(t))
        finally:
            c.close()
        if kind == cref.EV_REJECT:
            assert ref[1][0] == 0


@pytest.mark.parametrize("win", (7, 32))
def test_epsilon_at_a_logged_step(scenes, win):
    """lk_epsilon with epsilon^2 the first double at or above a logged level-0 step's |delta|^2 ends the solve on that
    step; the double below lets it go on."""
    from oracle import cref
    a, b, pts = scenes["noise"]
    log = _log(a, b, pts, win)
    found = 0
    for ev in log[(log["kind"] == cref.EV_EPS) & (log["level"] == 0)][:200]:
        d2 = float(ev["d2"])
        e = float(np.sqrt(d2))
        while e * e < d2:
            e = float(np.nextafter(e, np.inf))
        while float(np.nextafter(e, 0.0)) ** 2 >= d2:
            e = float(np.nextafter(e, 0.0))
        e_lo = float(np.nextafter(e, 0.0))
        p = pts[ev["pt"]:ev["pt"] + 1]
        hi, lo = _log(a, b, p, win, epsilon=e), _log(a, b, p, win, epsilon=e_lo)
        sel = lambda lg: lg[(lg["level"] == 0) & (lg["iter"] == ev["iter"]) & (lg["d2"] == d2)]
        if not (len(sel(hi)) and sel(hi)["kind"][0] == cref.EV_EPS and len(sel(lo)) and sel(lo)["kind"][0] != cref.EV_EPS):
            continue                        # the new epsilon changed the path before this step
        for eps in (e, e_lo):
            c = _context(win, lk_epsilon=eps)
            try:
                _check_track(c, a, b, p, win, f"W={win} epsilon={eps!r}", epsilon=eps)
            finally:
                c.close()
        found += 1
        if found == 3:
            break
    assert found >= 1


# ----------------------------------------------------------------------------- the modes
def _reference_unit(u, n_select, t_prev, win):
    """test_gpu_path.reference_unit (cv2) with a win x win window"""
    from oracle import ref_path
    corners = ref_path.fast_cv2(u["l0"])
    pts = synth.select_features(corners, n_select)
    fs = ref_path.FeatureSet(); fs.points = pts.copy(); fs.ages = np.zeros(len(pts), np.int32)
    cm = S.circular_matching(u["l0"], u["r0"], u["l1"], u["r1"], pts, fs, win)
    ok = ref_path.check_valid_match(cm["l0"], cm["l0_ret"], 0)
    pL0, pR0, pL1, pR1 = (ref_path.remove_invalid_points(cm[k], ok) for k in ("l0", "r0", "l1", "r1"))
    X = ref_path.triangulate(u["P_l"], u["P_r"], pL0, pR0, "cv2")
    R, t, inl, _ = ref_path.tracking_frame2frame(u["P_l"], pL0, pL1, X, t_prev, "cv2")
    return dict(n_detected=len(corners), pts=pts, kept3=cm["kept_idx"], kept=cm["kept_idx"][ok], l0=pL0, r0=pR0, l1=pL1,
                r1=pR1, X=X, R=R, t=t, inliers=inl)


BATCH_CONFIGS = {"graphs-partition0": dict(graphs=1, sm_partition=0), "graphs-partition8": dict(graphs=1, sm_partition=8),
                 "plain-partition0": dict(graphs=0, sm_partition=0), "plain-partition8": dict(graphs=0, sm_partition=8)}
T_PREV = (0.0, 0.0, -0.8)


@pytest.mark.parametrize("win", MODE_WINDOWS)
def test_batched_modes(built, win):
    units = [synth.stereo_unit(1241, 376, 60 + i) for i in range(4)]
    refs = [_reference_unit(u, 2000, np.array(T_PREV), win) for u in units]
    for name, opts in BATCH_CONFIGS.items():
        c = _context(win, opts)
        try:
            c.batch_configure(1241, 376, 8, units[0]["P_l"], units[0]["P_r"])
            arr, keep, pitch = c.make_units([dict(u, n_select=2000, t_prev=T_PREV) for u in units])
            res = c.frame_batch(arr, pitch)
            for i, ref in enumerate(refs):
                check_unit(res[i], c.batch_fetch(i, res[i]), ref)
            c.batch_submit(arr, 4, pitch)
            res = c.batch_wait(4, 4)
            for i, ref in enumerate(refs):
                check_unit(res[i], c.batch_fetch(4 + i, res[i]), ref)
        except AssertionError as e:
            raise AssertionError(f"W={win} {name}: {e}") from e
        finally:
            c.close()
    assert all(len(r["kept"]) > 0 for r in refs)


def _drive(w, h, seed, n):
    base = synth.stereo_unit(w, h, seed)
    fr = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=synth.SEQ_STEP_R * k, tvec=synth.SEQ_STEP_T * k)
        fr.append((u["l1"], u["r1"]))
    return base["P_l"], base["P_r"], fr


def _seq_push_run(c, P_l, P_r, frames):
    c.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    out = []
    for k in range(1, len(frames)):
        out.append(c.seq_push(*frames[k]))
        out[-1]["pose"] = c.seq_pose()
        out[-1]["state"] = c.seq_state()
    return out


@pytest.mark.parametrize("win", MODE_WINDOWS)
def test_sequence_mode_against_the_reference_glue(built, win):
    """vo_seq_push over 12 frames: point lists and the carried FeatureSet exact, [R|t] within 1e-8 of cv2's, frame_pose
    as integrated from them"""
    from oracle import ref_path
    P_l, P_r, frames = _drive(1241, 376, 31, 13)
    c = _context(win, max_features=8192)
    try:
        got = _seq_push_run(c, P_l, P_r, frames)
    finally:
        c.close()
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    for k in range(1, len(frames)):
        (l0, r0), (l1, r1) = frames[k - 1], frames[k]
        g, where = got[k - 1], f"W={win} frame {k}"
        pL0, pR0, pL1, pR1, info = S.matching_features(l0, r0, l1, r1, fs, win)
        assert g["n_features"] == len(info["bucketed"]) and g["n_tracked"] == len(info["kept_idx"]), where
        for name, ref in (("l0", pL0), ("r0", pR0), ("l1", pL1), ("r1", pR1)):
            assert np.array_equal(g[name], ref), f"{where}: {name}"
        pts, ages, _ = g["state"]
        assert np.array_equal(pts, fs.points) and np.array_equal(ages, fs.ages), f"{where}: carried FeatureSet"
        assert len(pL0) >= 4, where
        X = ref_path.triangulate(P_l, P_r, pL0, pR0, "cv2")
        R, translation, inl, _ = ref_path.tracking_frame2frame(P_l, pL0, pL1, X, translation, "cv2")
        assert g["n_inliers"] == len(inl), where
        assert max(np.abs(g["R"] - R).max(), np.abs(g["tvec"] - translation).max()) <= POSE_TOL, where
        frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
        assert np.abs(g["pose"] - frame_pose).max() <= 1e-6 * max(1.0, np.abs(frame_pose).max()), f"{where}: frame_pose"


@pytest.mark.parametrize("win", MODE_WINDOWS)
def test_mseq_two_sizes_each_as_run_alone(built, win):
    """640 x 240 and 600 x 232 (the same pyramid depth at each of these windows) through vo_mseq_begin_sized"""
    from oracle import cref
    drives = [_drive(640, 240, 31, 6), _drive(600, 232, 8, 6)]
    assert len({cref.Pyramid(d[2][0][0], win).nlevels() for d in drives}) == 1
    P_l = np.stack([d[0] for d in drives]); P_r = np.stack([d[1] for d in drives])
    c = _context(win, max_features=8192)
    try:
        alone = [_seq_push_run(c, P_l[q], P_r[q], drives[q][2]) for q in range(2)]
        c.mseq_begin([d[2][0][0] for d in drives], [d[2][0][1] for d in drives], P_l, P_r)
        for k in range(1, 6):
            c.mseq_submit([d[2][k][0] for d in drives], [d[2][k][1] for d in drives])
            recs = c.mseq_wait()
            for q in range(2):
                _same(recs[q], alone[q][k - 1], f"W={win} sequence {q} frame {k}")
                assert np.array_equal(c.mseq_pose(q), alone[q][k - 1]["pose"])
    finally:
        c.close()
    assert all(a[-1]["n_valid"] > 0 for a in alone)


@pytest.mark.parametrize("win", MODE_WINDOWS)
def test_frames_in_gpu_memory_equal_host_frames(built, win):
    torch = pytest.importorskip("torch")
    P_l, P_r, frames = _drive(1241, 376, 7, 6)
    dev = [(torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda()) for l, r in frames]
    c = _context(win, max_features=8192)
    try:
        host = _seq_push_run(c, P_l, P_r, frames)
        c.seq_begin_device(dev[0][0], dev[0][1], P_l, P_r)
        for k in range(1, len(frames)):
            _same(c.seq_push_device(*dev[k]), host[k - 1], f"W={win} device frame {k}")
        assert np.array_equal(c.seq_pose(), host[-1]["pose"])
    finally:
        c.close()
