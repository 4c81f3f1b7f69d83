"""Several independent sequences through the streaming sequence mode (vo_mseq_*): each sequence's records, point lists,
carried state and frame_pose are bit for bit those of running it alone through vo_seq_*, one sequence is anchored to the
reference path (cv2), and pipelining, colour input, retirement, a textureless frame, the launch count and every refusal
are covered."""
import ctypes as C

import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

W, H, NF = 640, 240, 12
# five drives: (seed, per-frame rotation, per-frame translation)
DRIVES = [
    (31, (0.001, -0.004, 0.0005), (0.01, -0.003, -0.2)),
    (7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25)),
    (13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15)),
    (42, (0.003, -0.001, 0.0005), (0.015, 0.0, -0.3)),
    (5, (-0.001, -0.002, 0.001), (0.0, -0.005, -0.18)),
]
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
ARRAYS = ("rvec", "tvec", "R", "l0", "r0", "l1", "r1")


def _drive(seed, r, t, n=NF, w=W, h=H):
    base = synth.stereo_unit(w, h, seed)
    out = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=np.array(r) * k, tvec=np.array(t) * k)
        out.append((u["l1"], u["r1"]))
    return base, out


@pytest.fixture(scope="module")
def drives():
    d = [_drive(*x) for x in DRIVES]
    return d[0][0]["P_l"], d[0][0]["P_r"], [fr for _, fr in d]


def _same(a, b, where):
    for k in INTS:
        assert a[k] == b[k], f"{where}: {k} {a[k]} != {b[k]}"
    for k in ARRAYS:
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), f"{where}: {k}"


def _run_mseq(ctx, P_l, P_r, frames, pipelined=False, edit=None):
    """frames[q][k] = (left, right); edit(q, k, pair) -> pair lets a test change or retire (None, None) a frame.
    Returns per frame: (records, [state of q], [pose of q]) -- state / pose only for submit-then-wait runs."""
    n = len(frames)
    pair = (lambda q, k: frames[q][k]) if edit is None else (lambda q, k: edit(q, k, frames[q][k]))
    ctx.mseq_begin([frames[q][0][0] for q in range(n)], [frames[q][0][1] for q in range(n)], P_l, P_r)
    out = []

    def submit(k):
        ps = [pair(q, k) for q in range(n)]
        ctx.mseq_submit([p[0] for p in ps], [p[1] for p in ps])

    if pipelined:
        submit(1)
        for k in range(1, NF):
            if k + 1 < NF:
                submit(k + 1)
            out.append((ctx.mseq_wait(), None, None))
        return out
    for k in range(1, NF):
        submit(k)
        recs = ctx.mseq_wait()
        out.append((recs, [ctx.mseq_state(q) for q in range(n)], [ctx.mseq_pose(q) for q in range(n)]))
    return out


@pytest.fixture(scope="module")
def mseq_run(ctx, drives):
    P_l, P_r, frames = drives
    return _run_mseq(ctx, P_l, P_r, frames)


def test_each_sequence_is_bit_identical_to_running_it_alone(ctx, drives, mseq_run):
    from visual_odom_b200 import capi
    P_l, P_r, frames = drives
    for q, fr in enumerate(frames):
        ctx.seq_begin(fr[0][0], fr[0][1], P_l, P_r)
        for k in range(1, NF):
            alone = ctx.seq_push(*fr[k])
            recs, states, poses = mseq_run[k - 1]
            assert recs[q]["status"] == capi.VO_OK
            _same(recs[q], alone, f"sequence {q} frame {k}")
            st = ctx.seq_state()
            for name, a, b in zip(("points", "ages", "translation"), states[q], st):
                assert a.dtype == b.dtype and np.array_equal(a, b), f"sequence {q} frame {k}: carried {name}"
            assert np.array_equal(poses[q], ctx.seq_pose()), f"sequence {q} frame {k}: frame_pose"
        assert alone["n_valid"] > 50 and alone["n_inliers"] > 20
        assert np.linalg.norm(ctx.seq_pose()[:3, 3]) > 0.5            # the drive actually advanced


def test_one_sequence_matches_the_reference_path(drives, mseq_run):
    """Sequence 0 of the batched run, frame by frame against cv2 through the reference's glue (oracle/ref_path.py)."""
    pytest.importorskip("cv2")
    from oracle import ref_path
    P_l, P_r, frames = drives
    fr = frames[0]
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    for k in range(1, NF):
        (l0, r0), (l1, r1) = fr[k - 1], fr[k]
        recs, states, poses = mseq_run[k - 1]
        got = recs[0]
        pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend="cv2")
        X = ref_path.triangulate(P_l, P_r, pL0, pR0, "cv2")
        R, translation, inl, rvec = ref_path.tracking_frame2frame(P_l, pL0, pL1, X, translation, "cv2")
        assert got["n_features"] == len(info["bucketed"]) and got["n_tracked"] == len(info["kept_idx"])
        assert got["n_valid"] == len(pL0)
        for name, ref in (("l0", pL0), ("r0", pR0), ("l1", pL1), ("r1", pR1)):
            assert np.array_equal(got[name], ref), f"frame {k}: {name}"
        assert got["n_inliers"] == len(inl), f"frame {k}: inlier count"
        assert np.linalg.norm(got["R"] - R) / np.linalg.norm(R) <= 1e-4
        assert np.linalg.norm(got["tvec"] - translation) / np.linalg.norm(translation) <= 1e-4
        frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
        assert np.abs(poses[0] - frame_pose).max() <= 1e-6 * max(1.0, np.abs(frame_pose).max()), f"frame {k}: frame_pose"
        pts, ages, _ = states[0]
        assert np.array_equal(pts, fs.points) and np.array_equal(ages, fs.ages), f"frame {k}: carried FeatureSet"


def test_two_submissions_in_flight_equal_submit_then_wait(ctx, drives, mseq_run):
    P_l, P_r, frames = drives
    got = _run_mseq(ctx, P_l, P_r, frames, pipelined=True)
    for k, ((a, _, _), (b, states, poses)) in enumerate(zip(got, mseq_run), start=1):
        for q in range(len(frames)):
            _same(a[q], b[q], f"sequence {q} frame {k}")
    for q in range(len(frames)):
        assert np.array_equal(ctx.mseq_pose(q), mseq_run[-1][2][q])
        assert all(np.array_equal(x, y) for x, y in zip(ctx.mseq_state(q), mseq_run[-1][1][q]))


def test_bgr_input_equals_gray_input(ctx, drives, mseq_run):
    """B = G = R = gray converts back to the same gray plane (cv::cvtColor's weights sum to 2^15)."""
    P_l, P_r, frames = drives
    bgr = [[(np.repeat(l[:, :, None], 3, 2), np.repeat(r[:, :, None], 3, 2)) for l, r in fr] for fr in frames]
    got = _run_mseq(ctx, P_l, P_r, bgr)
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(got, mseq_run), start=1):
        for q in range(len(frames)):
            _same(a[q], b[q], f"sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q])
            assert all(np.array_equal(x, y) for x, y in zip(sa[q], sb[q]))


def test_a_textureless_or_retired_sequence_leaves_the_others_alone(ctx, drives, mseq_run):
    from visual_odom_b200 import capi
    P_l, P_r, frames = drives
    flat, gone, k_flat, k_gone = 1, 3, 4, 6
    blank = np.full((H, W), 128, np.uint8)

    def edit(q, k, pair):
        if q == flat and k in (k_flat, k_flat + 1):
            return blank, blank
        if q == gone and k >= k_gone:
            return None, None
        return pair

    got = _run_mseq(ctx, P_l, P_r, frames, edit=edit)
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(got, mseq_run), start=1):
        for q in range(len(frames)):
            if q == flat and k >= k_flat:
                continue
            if q == gone and k >= k_gone:
                assert a[q]["status"] == capi.VO_MSEQ_RETIRED and a[q]["n_features"] == 0, f"frame {k}"
                # frozen at what its last frame (k_gone - 1, list index k_gone - 2) left
                _, s_last, p_last = mseq_run[k_gone - 2]
                assert np.array_equal(pa[q], p_last[q]), f"frame {k}: frozen frame_pose"
                assert all(np.array_equal(x, y) for x, y in zip(sa[q], s_last[q])), f"frame {k}: frozen state"
                continue
            _same(a[q], b[q], f"sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q]) and all(np.array_equal(x, y) for x, y in zip(sa[q], sb[q]))
    # (got[k - 1] is frame k) the first flat pair: nothing survives the circular check on it; the second: FAST finds no
    # corner on the flat previous image and nothing was carried, so the frame has no features at all
    first = got[k_flat - 1][0][flat]
    assert first["n_valid"] == 0 and first["pnp_status"] == capi.VO_E_TOO_FEW_POINTS
    after = got[k_flat][0][flat]
    assert after["status"] == capi.VO_OK and after["n_features"] == 0 and after["pnp_status"] == capi.VO_E_TOO_FEW_POINTS
    # a retired sequence cannot come back
    n = len(frames)
    with pytest.raises(RuntimeError, match="was retired"):
        ctx.mseq_submit([f[1][0] for f in frames], [f[1][1] for f in frames])
    # everything retired: submissions still work and report only retirements
    ctx.mseq_submit([None] * n, [None] * n)
    assert all(r["status"] == capi.VO_MSEQ_RETIRED for r in ctx.mseq_wait())


def test_launches_per_submission_do_not_grow_with_the_sequence_count(built):
    from visual_odom_b200.capi import Context
    w, h = 320, 120
    base, fr = _drive(3, *DRIVES[0][1:], n=6, w=w, h=h)
    c = Context(0, max_features=1024)

    def per_submission(n):
        c.mseq_begin([fr[0][0]] * n, [fr[0][1]] * n, base["P_l"], base["P_r"])
        for k in (1, 2):                      # captures the graphs of both buffer parities
            c.mseq_submit([fr[k][0]] * n, [fr[k][1]] * n); c.mseq_wait(want_points=False)
        l0 = c.kernel_launches()
        for k in range(3, 6):
            c.mseq_submit([fr[k][0]] * n, [fr[k][1]] * n); c.mseq_wait(want_points=False)
        return (c.kernel_launches() - l0) / 3

    one, sixteen = per_submission(1), per_submission(16)
    c.seq_begin(fr[0][0], fr[0][1], base["P_l"], base["P_r"])
    for k in (1, 2):
        c.seq_push(*fr[k])
    l0 = c.kernel_launches()
    for k in range(3, 6):
        c.seq_push(*fr[k])
    alone = (c.kernel_launches() - l0) / 3
    assert one == sixteen == alone and one > 0
    c.close()


def test_misuse_is_refused_and_the_context_stays_usable(ctx, drives, mseq_run):
    from visual_odom_b200 import capi
    P_l, P_r, frames = drives
    n = len(frames)
    L = [fr[0][0] for fr in frames]; R = [fr[0][1] for fr in frames]

    def code(fn):
        with pytest.raises(capi.VoError) as e:
            fn()
        return e.value.code

    assert code(lambda: ctx.mseq_begin([], [], P_l, P_r)) == capi.VO_E_INVALID
    assert code(lambda: ctx.mseq_begin([L[0]] * (capi.VO_MSEQ_MAX + 1), [R[0]] * (capi.VO_MSEQ_MAX + 1), P_l, P_r)) == capi.VO_E_CAPACITY
    ctx.set_option("mono_rotation", 1)
    try:
        assert code(lambda: ctx.mseq_begin(L, R, P_l, P_r)) == capi.VO_E_UNSUPPORTED
    finally:
        ctx.set_option("mono_rotation", 0)
    ctx.mseq_begin(L, R, P_l, P_r)
    assert code(lambda: ctx.mseq_wait()) == capi.VO_E_INVALID                     # nothing in flight
    # one image of a pair NULL (the C call directly: the binding refuses it before)
    lp, rp = (C.c_void_p * n)(), (C.c_void_p * n)()
    for q in range(n):
        lp[q], rp[q] = frames[q][1][0].ctypes.data, frames[q][1][1].ctypes.data
    rp[2] = None
    assert ctx.lib.vo_mseq_submit(ctx.h, lp, rp, W, 1) == capi.VO_E_INVALID
    # the single-sequence frame calls are refused while vo_mseq_* sequences run
    assert code(lambda: ctx.seq_push(frames[0][1][0], frames[0][1][1])) == capi.VO_E_INVALID
    assert code(lambda: ctx.seq_pose()) == capi.VO_E_INVALID
    for k in (1, 2):
        ctx.mseq_submit([fr[k][0] for fr in frames], [fr[k][1] for fr in frames])
    assert code(lambda: ctx.mseq_submit([fr[3][0] for fr in frames], [fr[3][1] for fr in frames])) == capi.VO_E_INVALID
    # while submissions are in flight: another sequence mode and the host-buffer calls are refused
    assert code(lambda: ctx.seq_begin(L[0], R[0], P_l, P_r)) == capi.VO_E_INVALID
    assert code(lambda: ctx.fast_detect(L[0])) == capi.VO_E_INVALID
    for k in (1, 2):                               # and the run goes on as if nothing had happened
        recs = ctx.mseq_wait()
        for q in range(n):
            _same(recs[q], mseq_run[k - 1][0][q], f"sequence {q} frame {k}")
    assert code(lambda: ctx.mseq_wait()) == capi.VO_E_INVALID
    assert code(lambda: ctx.mseq_pose(n)) == capi.VO_E_INVALID
    # an idle multi-sequence run is ended by vo_seq_begin, whose sequence then works as usual
    ctx.seq_begin(L[0], R[0], P_l, P_r)
    assert code(lambda: ctx.mseq_pose(0)) == capi.VO_E_INVALID
    _same(ctx.seq_push(*frames[0][1]), mseq_run[0][0][0], "sequence 0 alone")
