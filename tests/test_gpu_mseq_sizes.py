"""Sequences of different image sizes in one multi-sequence context (vo_mseq_begin_sized): every sequence is bit for bit
what it gives when run alone through vo_seq_* at its own size and calibration, in both buffer parities, with the
mono_rotation branch, under reordering, pipelining, graphs on or off, colour input and retirement of the largest sequence;
one sequence is anchored to cv2; a plane that held a larger image before holds no stale derivatives; one size repeated is
vo_mseq_begin_calib exactly, at the same launch count; and every refusal leaves the context usable."""
import ctypes as C

import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

K0 = synth.KITTI00
NF = 5                      # frames 0 .. 4: four submissions, both buffer parities twice


def _cal(sx=1.0, sy=1.0, dcx=0.0, dcy=0.0, sb=1.0):
    return dict(fx=K0["fx"] * sx, fy=K0["fy"] * sy, cx=K0["cx"] + dcx, cy=K0["cy"] + dcy, bf=K0["bf"] * sb)


# (w, h, seed, per-frame rotation, per-frame translation, calibration)
# the three image sizes of the KITTI odometry training sequences (00-02, 03, 04-10)
KITTI = [
    (1241, 376, 3, (0.001, 0.002, 0.0), (0.01, 0.0, -0.22), _cal(1.1, 1.1, 0.0, 0.0, 0.85)),
    (1242, 375, 11, (-0.002, -0.001, 0.0005), (0.0, 0.003, -0.2), _cal(0.9, 0.9, -30.0, 12.0)),
    (1226, 370, 19, (0.0, -0.003, 0.001), (-0.01, 0.0, -0.26), _cal(1.0, 1.0, 35.0, -20.0, 1.15)),
]
# smaller sizes of the same pyramid depth, odd widths and heights among them; the 512 x 200 drive pans (rotation about
# the vertical and horizontal axes) so that its tracks leave through the right and bottom edges
SMALL = [
    (640, 240, 31, (0.001, -0.004, 0.0005), (0.01, -0.003, -0.2), _cal()),
    (601, 233, 7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25), _cal(0.9, 0.9, -300.0, -60.0)),
    (656, 248, 13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15), _cal(1.1, 1.1, -280.0, -55.0)),
    (512, 200, 42, (-0.006, 0.012, 0.0005), (0.03, 0.01, -0.3), _cal(1.0, 1.0, -350.0, -85.0, 1.15)),
]
INTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
ARRAYS = ("rvec", "tvec", "R", "l0", "r0", "l1", "r1")


def _group(drives):
    P_l, P_r, frames = [], [], []
    for w, h, seed, r, t, cal in drives:
        base = synth.stereo_unit(w, h, seed, cal=cal)
        fr = [(base["l0"], base["r0"])]
        for k in range(1, NF):
            u = synth.stereo_unit(w, h, seed, cal=cal, rvec=np.array(r) * k, tvec=np.array(t) * k)
            fr.append((u["l1"], u["r1"]))
        P_l.append(base["P_l"]); P_r.append(base["P_r"]); frames.append(fr)
    return np.stack(P_l), np.stack(P_r), frames


@pytest.fixture(scope="module", params=["kitti", "small"])
def group(request):
    return _group(KITTI if request.param == "kitti" else SMALL)


@pytest.fixture(scope="module")
def small():
    return _group(SMALL)


def _context():
    from visual_odom_b200.capi import Context
    return Context(0, max_features=8192)                # as the shared context


@pytest.fixture(scope="module")
def small_alone(built, small):
    """Each small drive through vo_seq_* on a context of its own: per sequence, per frame (record, state, pose)."""
    P_l, P_r, frames = small
    out = []
    for q, fr in enumerate(frames):
        c = _context()
        out.append(_alone(c, P_l[q], P_r[q], fr))
        c.close()
    return out


def _same(a, b, where, keys=ARRAYS):
    for k in INTS:
        assert a[k] == b[k], f"{where}: {k} {a[k]} != {b[k]}"
    for k in keys:
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), f"{where}: {k}"


def _run_mseq(ctx, P_l, P_r, frames, pipelined=False, mono=False, retire=None, bgr=False):
    """Per frame: (records, [state of q], [pose of q]); state / pose only for submit-then-wait runs.  retire = (q, k):
    sequence q gets a NULL pair from frame k on.  bgr: every image as 3-channel BGR (b = g = r)."""
    n = len(frames)
    img = (lambda a: np.repeat(a[:, :, None], 3, axis=2)) if bgr else (lambda a: a)
    ctx.mseq_begin([img(f[0][0]) for f in frames], [img(f[0][1]) for f in frames], P_l, P_r, mono_rotation=mono)

    def submit(k):
        ps = [(None, None) if retire and q == retire[0] and k >= retire[1] else (img(frames[q][k][0]), img(frames[q][k][1]))
              for q in range(n)]
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
    """vo_seq_begin / vo_seq_push of one sequence at its own size with its own matrices: per frame (record, state, pose)."""
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


def _check_against(run, alone, mono=False, skip=()):
    from visual_odom_b200 import capi
    for q, ref in enumerate(alone):
        if q in skip:
            continue
        for k, ((recs, states, poses), (rec, st, pose)) in enumerate(zip(run, ref), start=1):
            assert recs[q].get("status", capi.VO_OK) == capi.VO_OK       # vo_seq_* records carry none (errors raise)
            _same(recs[q], rec, f"sequence {q} frame {k}")
            if mono:
                for key in ("status", "n_inliers", "ransac_iters", "n_good"):
                    assert recs[q]["mono"][key] == rec["mono"][key], f"sequence {q} frame {k}: mono {key}"
                for key in ("R", "t"):
                    assert np.array_equal(recs[q]["mono"][key], rec["mono"][key]), f"sequence {q} frame {k}: mono {key}"
                assert np.array_equal(recs[q]["ess_mask"], rec["ess_mask"]), f"sequence {q} frame {k}: essential mask"
            if states is not None:
                for name, a, b in zip(("points", "ages", "translation"), states[q], st):
                    assert a.dtype == b.dtype and np.array_equal(a, b), f"sequence {q} frame {k}: carried {name}"
                assert np.array_equal(poses[q], pose), f"sequence {q} frame {k}: frame_pose"
        assert ref[-1][0]["n_valid"] > 30 and ref[-1][0]["n_inliers"] > 10


def _alone_all(ctx, P_l, P_r, frames, mono=False):
    return [_alone(ctx, P_l[q], P_r[q], fr, mono) for q, fr in enumerate(frames)]


def test_each_sequence_is_bit_identical_to_running_it_alone_at_its_size(ctx, group):
    P_l, P_r, frames = group
    assert len({f[0][0].shape for f in frames}) == len(frames)
    run = _run_mseq(ctx, P_l, P_r, frames)
    _check_against(run, _alone_all(ctx, P_l, P_r, frames))
    # the unequal FeatureSet lengths (points vs ages) are carried per sequence as well
    assert any(len(s[0]) != len(s[1]) for s in run[-1][1])


def test_mono_branch_is_bit_identical_to_running_it_alone_at_its_size(ctx, small):
    P_l, P_r, frames = small
    run = _run_mseq(ctx, P_l, P_r, frames, mono=True)
    _check_against(run, _alone_all(ctx, P_l, P_r, frames, mono=True), mono=True)


def test_tracks_leave_the_small_panning_drive_through_its_right_and_bottom_edges(small_alone):
    """The panning drive moves the image content right and down by about 9 and 5 pixels a frame, so tracks cross the
    right and bottom edges, where the LK ring's image bounds, the border and the bucket grid of its own size decide."""
    q = 3
    w, h = SMALL[q][0], SMALL[q][1]
    for rec, _, _ in small_alone[q]:
        d = (rec["l1"] - rec["l0"]).mean(axis=0)
        assert d[0] > 5 and d[1] > 2
        assert rec["n_tracked"] < rec["n_features"]
    allpts = np.concatenate([r[0]["l1"] for r in small_alone[q]])
    assert allpts[:, 0].max() > w - 10 and allpts[:, 1].max() > h - 10


def test_a_sequence_neither_first_nor_largest_matches_the_reference_path(ctx, small):
    """Sequence 1 (601 x 233) frame by frame against cv2 through the reference's glue (oracle/ref_path.py)."""
    pytest.importorskip("cv2")
    from oracle import ref_path
    P_l, P_r, frames = small
    run = _run_mseq(ctx, P_l, P_r, frames)
    q = 1
    assert frames[q][0][0].size < max(f[0][0].size for f in frames)
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


def test_a_plane_that_held_a_larger_image_holds_no_stale_derivatives(small, small_alone):
    """One context: a run with the 656 x 248 drive in sequence 0's planes, then, in the same envelope, a run with the
    panning 512 x 200 drive there (its LK windows at the right and bottom edges read the derivative band the larger image
    wrote).  Then vo_seq_* and the batched mode at the envelope size, which reuse the planes, equal fresh contexts."""
    P_l, P_r, frames = small
    big, pan = 2, 3
    c = _context()
    first = _run_mseq(c, P_l[[big, pan]], P_r[[big, pan]], [frames[big], frames[pan]])
    _check_against(first, [small_alone[big], small_alone[pan]])
    second = _run_mseq(c, P_l[[pan, big]], P_r[[pan, big]], [frames[pan], frames[big]])
    _check_against(second, [small_alone[pan], small_alone[big]])
    # a single sequence at the envelope size on the same planes = on a fresh context
    fr = frames[big]
    reused = _alone(c, P_l[big], P_r[big], fr)
    _check_against([([r], [st], [pose]) for r, st, pose in reused], [small_alone[big]])     # records, carried state, pose
    # the batched mode at the envelope size, on the same planes = on a fresh context
    W, H = fr[0][0].shape[1], fr[0][0].shape[0]
    u = synth.stereo_unit(W, H, 77)
    units = [dict(l0=u["l0"], r0=u["r0"], l1=u["l1"], r1=u["r1"], n_select=1500)] * 2

    def batch(cc):
        cc.set_option("batch_outputs", 1)
        cc.batch_configure(W, H, 2, u["P_l"], u["P_r"])
        arr, keep, pitch = cc.make_units(units)
        cc.batch_submit(arr, 0, pitch)
        recs = cc.batch_wait(0, 2)
        return [(r, cc.batch_outputs(i, r)) for i, r in enumerate(recs)]

    # the batched run after a mixed run on this context's planes
    _run_mseq(c, P_l[[pan, big]], P_r[[pan, big]], [frames[pan], frames[big]])
    got = batch(c)
    c.close()
    f = _context()
    ref = batch(f)
    f.close()
    for i in range(2):
        _same(got[i][0], ref[i][0], f"batched unit {i}", keys=("rvec", "tvec", "R"))
        for k in ("l0", "r0", "l1", "r1", "kept_idx", "X", "inliers"):
            assert np.array_equal(got[i][1][k], ref[i][1][k]), f"batched unit {i}: {k}"


# a second set of sizes in the envelope of {656 x 248, 512 x 200} whose bucket grid is larger: 656 x 200 has
# (200/20 + 1) x (656/20 + 1) = 363 cells against the 308 of 656 x 248, and its drive buckets more than 308 features
REGRID = [
    (656, 200, 13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15), _cal(1.1, 1.1, -280.0, -85.0)),
    (512, 248, 42, (0.001, -0.003, 0.0005), (0.01, 0.0, -0.2), _cal(1.0, 1.0, -350.0, -60.0)),
]


def test_a_larger_bucket_grid_in_the_same_envelope_tracks_every_feature(small, small_alone):
    """The front stage's captured graph holds the LK launch bound (the largest bucket grid of the sizes).  A later set of
    sizes with the same envelope but a larger grid must not replay a graph that leaves its extra features unsolved."""
    P_l, P_r, frames = small
    Pl2, Pr2, frames2 = _group(REGRID)
    alone2 = []
    for q, fr in enumerate(frames2):
        f = _context()
        alone2.append(_alone(f, Pl2[q], Pr2[q], fr))
        f.close()
    assert max(r[0]["n_features"] for r in alone2[0]) > 308
    c = _context()
    try:
        for graphs in (1, 0):
            c.set_option("graphs", graphs)
            first = _run_mseq(c, P_l[[2, 3]], P_r[[2, 3]], [frames[2], frames[3]])           # envelope 656 x 248
            _check_against(first, [small_alone[2], small_alone[3]])
            second = _run_mseq(c, Pl2, Pr2, frames2)                                          # same envelope
            _check_against(second, alone2)
    finally:
        c.close()


def test_order_pipelining_graphs_colour_and_retiring_the_largest(ctx, small, small_alone):
    from visual_odom_b200 import capi
    P_l, P_r, frames = small
    n = len(frames)
    ref = _run_mseq(ctx, P_l, P_r, frames)
    _check_against(ref, small_alone)
    # reversing the sequences (with their calibrations and sizes) reverses the results
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
    # BGR input (b = g = r, which cvtColor maps back to the gray value) = gray input
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(_run_mseq(ctx, P_l, P_r, frames, bgr=True), ref), start=1):
        for q in range(n):
            _same(a[q], b[q], f"BGR: sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q]) and all(np.array_equal(x, y) for x, y in zip(sa[q], sb[q]))
    # retiring the largest sequence (the one that sets the envelope) leaves the others bit-identical
    gone = int(np.argmax([f[0][0].size for f in frames]))
    k_gone = 2
    ret = _run_mseq(ctx, P_l, P_r, frames, retire=(gone, k_gone))
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(ret, ref), start=1):
        for q in range(n):
            if q == gone and k >= k_gone:
                assert a[q]["status"] == capi.VO_MSEQ_RETIRED
                continue
            _same(a[q], b[q], f"retired {gone}: sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q]) and all(np.array_equal(x, y) for x, y in zip(sa[q], sb[q]))


def _ptrs(pairs):
    n = len(pairs)
    return [p[0].ctypes.data for p in pairs], [p[1].ctypes.data for p in pairs]


def test_one_size_repeated_is_begin_calib_bit_for_bit_and_at_the_same_launch_count(ctx, small):
    P_l, P_r, frames = small
    frames = [frames[0]] * 3                           # one size (640 x 240) for all
    P_l, P_r = P_l[:3], P_r[:3]
    n = len(frames)
    w, h = frames[0][0][0].shape[1], frames[0][0][0].shape[0]

    def run(sized):
        lp, rp = _ptrs([f[0] for f in frames])
        if sized:
            ctx.mseq_begin_ptr([w] * n, [h] * n, lp, rp, [w] * n, P_l, P_r)
        else:
            ctx.mseq_begin_ptr(w, h, lp, rp, w, P_l, P_r)
        out = []
        l0 = None
        for k in range(1, NF):
            if k == 3:
                l0 = ctx.kernel_launches()
            lp, rp = _ptrs([f[k] for f in frames])
            if sized:
                ctx.mseq_submit_ptr(lp, rp, [w] * n)
            else:
                ctx.mseq_submit_ptr(lp, rp, w)
            recs = ctx.mseq_wait()
            out.append((recs, [ctx.mseq_state(q) for q in range(n)], [ctx.mseq_pose(q) for q in range(n)]))
        return out, (ctx.kernel_launches() - l0) / 2

    calib, lc = run(False)
    sized, ls = run(True)
    assert lc == ls and lc > 0
    for k, ((a, sa, pa), (b, sb, pb)) in enumerate(zip(sized, calib), start=1):
        for q in range(n):
            _same(a[q], b[q], f"sequence {q} frame {k}")
            assert np.array_equal(pa[q], pb[q]) and all(np.array_equal(x, y) for x, y in zip(sa[q], sb[q]))


def test_launches_per_submission_do_not_depend_on_the_count_or_the_sizes(built, small):
    P_l, P_r, frames = small
    c = _context()
    nd = len(frames)

    def per_submission(m):
        fr = [frames[q % nd] for q in range(m)]
        Pl = np.stack([P_l[q % nd] for q in range(m)]); Pr = np.stack([P_r[q % nd] for q in range(m)])
        c.mseq_begin([f[0][0] for f in fr], [f[0][1] for f in fr], Pl, Pr)
        for k in (1, 2):                      # captures the graphs of both buffer parities
            c.mseq_submit([f[k][0] for f in fr], [f[k][1] for f in fr]); c.mseq_wait(want_points=False)
        l0 = c.kernel_launches()
        for k in (3, 4):
            c.mseq_submit([f[k][0] for f in fr], [f[k][1] for f in fr]); c.mseq_wait(want_points=False)
        return (c.kernel_launches() - l0) / 2

    one, mixed16 = per_submission(1), per_submission(16)
    fr = frames[0]
    c.seq_begin(fr[0][0], fr[0][1], P_l[0], P_r[0])
    for k in (1, 2):
        c.seq_push(*fr[k])
    l0 = c.kernel_launches()
    for k in (3, 4):
        c.seq_push(*fr[k])
    alone = (c.kernel_launches() - l0) / 2
    c.close()
    assert one == mixed16 == alone and alone > 0


def test_refusals_leave_the_context_usable(ctx, small, small_alone):
    from visual_odom_b200 import capi
    P_l, P_r, frames = small
    n = len(frames)
    Pl = np.ascontiguousarray(P_l, np.float32); Pr = np.ascontiguousarray(P_r, np.float32)
    ws = np.array([f[0][0].shape[1] for f in frames], np.int32)
    hs = np.array([f[0][0].shape[0] for f in frames], np.int32)
    ps = ws.astype(np.uint64)
    lp, rp = (C.c_void_p * n)(), (C.c_void_p * n)()
    for q in range(n):
        lp[q], rp[q] = frames[q][0][0].ctypes.data, frames[q][0][1].ctypes.data
    lib, h = ctx.lib, ctx.h
    I, U = capi.VO_E_INVALID, capi.VO_E_UNSUPPORTED

    def begin(w=ws, hh=hs, p=ps, Pl_=Pl, Pr_=Pr, n_=n, l=lp, r=rp, ch=1, flags=0):
        arg = lambda a: None if a is None else a.ctypes.data
        return lib.vo_mseq_begin_sized(h, n_, arg(w), arg(hh), arg(Pl_), arg(Pr_), l, r, arg(p), ch, flags)

    def bad(i, a, v):
        a = a.copy(); a[i] = v
        return a

    assert begin(w=None) == I and begin(hh=None) == I and begin(p=None) == I
    assert begin(w=bad(1, ws, 0)) == I and begin(hh=bad(2, hs, -1)) == I
    assert begin(p=bad(3, ps, ws[3] - 1)) == I
    assert begin(ch=3) == I                                       # BGR needs 3 * w bytes per row
    assert begin(Pl_=None) == I and begin(Pr_=None) == I and begin(n_=0) == I and begin(flags=4) == I
    assert begin(n_=capi.VO_MSEQ_MAX + 1) == capi.VO_E_CAPACITY
    assert begin(hh=bad(0, hs, 9)) == U                           # rows / 10 == 0
    assert begin(w=bad(1, ws, 80)) == U                           # 80 wide: one pyramid level less
    err = lib.vo_last_error(h).decode()
    assert "80 x 233" in err and "640 x 240" in err, err
    # a single-pitch submission narrower than some live sequence, after a good begin
    ctx.mseq_begin_ptr(list(ws), list(hs), list(lp), list(rp), list(ps), Pl, Pr)
    W = int(ws.max())
    wide = [[np.zeros((hs[q], W), np.uint8) for _ in range(2)] for q in range(n)]     # frame 1 in rows of W bytes
    for q in range(n):
        for i in range(2):
            wide[q][i][:, :ws[q]] = frames[q][1][i]
    l1 = (C.c_void_p * n)(*[wide[q][0].ctypes.data for q in range(n)])
    r1 = (C.c_void_p * n)(*[wide[q][1].ctypes.data for q in range(n)])
    assert lib.vo_mseq_submit(h, l1, r1, W - 1, 1) == I
    assert lib.vo_mseq_submit_sized(h, l1, r1, None, 1) == I
    assert lib.vo_mseq_submit_sized(h, l1, r1, np.full(n, W, np.uint64).ctypes.data, 3) == I
    # and the context goes on: one pitch covering every width, then the rest of the drive, equals each sequence alone
    run = []
    for k in range(1, NF):
        if k == 1:
            assert lib.vo_mseq_submit(h, l1, r1, W, 1) == capi.VO_OK
        else:
            ctx.mseq_submit([frames[q][k][0] for q in range(n)], [frames[q][k][1] for q in range(n)])
        run.append((ctx.mseq_wait(), [ctx.mseq_state(q) for q in range(n)], [ctx.mseq_pose(q) for q in range(n)]))
    _check_against(run, small_alone)
