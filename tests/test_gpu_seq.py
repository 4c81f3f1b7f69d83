"""Streaming sequence mode (vo_seq_*): 20+ synthetic frames with the main-loop state (features, ages,
translation) resident on the GPU, compared frame by frame with the reference path (cv2 through the
verbatim glue of oracle/ref_path.py): FAST refill, bucketing (aliasing, overwrite rule), the carried
ages/points length skew, circular matching, triangulation, PnP with the carried extrinsic guess.
On this dense texture ages never pass 1, so neither the age limit of the buckets nor a stale age paired
with a fresh corner decides anything here: tests/test_gpu_long_tracks.py covers those on a sparse drive."""
import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

STEP_R = np.array([0.001, -0.004, 0.0005])
STEP_T = np.array([0.01, -0.003, -0.2])


def _frames(w, h, seed, n):
    base = synth.stereo_unit(w, h, seed)
    out = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=STEP_R * k, tvec=STEP_T * k)
        out.append((u["l1"], u["r1"]))
    return base, out


@pytest.mark.parametrize("w,h,nf", [(1241, 376, 22), (640, 480, 6)])
def test_sequence_state_carry_matches_reference(ctx, w, h, nf):
    pytest.importorskip("cv2")
    from oracle import ref_path
    base, frames = _frames(w, h, 31, nf)
    ctx.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    traj_ref, traj_gpu = [np.eye(4)], [np.eye(4)]
    for k in range(1, nf):
        l0, r0 = frames[k - 1]; l1, r1 = frames[k]
        got = ctx.seq_push(l1, r1)
        pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend="cv2")
        X = ref_path.triangulate(base["P_l"], base["P_r"], pL0, pR0, "cv2")
        R, translation, inl, rvec = ref_path.tracking_frame2frame(base["P_l"], pL0, pL1, X, translation, "cv2")
        assert got["n_features"] == len(info["bucketed"]), f"frame {k}: bucketed feature count"
        assert got["n_tracked"] == len(info["kept_idx"])
        assert got["n_valid"] == len(pL0)
        for name, ref in (("l0", pL0), ("r0", pR0), ("l1", pL1), ("r1", pR1)):
            assert np.array_equal(got[name], ref), f"frame {k}: {name}"
        assert got["n_inliers"] == len(inl), f"frame {k}: inlier count"
        assert np.linalg.norm(got["R"] - R) / np.linalg.norm(R) <= 1e-4
        assert np.linalg.norm(got["tvec"] - translation) / np.linalg.norm(translation) <= 1e-4
        frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
        assert np.abs(ctx.seq_pose() - frame_pose).max() <= 1e-6 * max(1.0, np.abs(frame_pose).max()), f"frame {k}: frame_pose"
        traj_ref.append(frame_pose.copy()); traj_gpu.append(ctx.seq_pose())
        pts, ages, t = ctx.seq_state()
        assert np.array_equal(pts, fs.points) and np.array_equal(ages, fs.ages), f"frame {k}: carried FeatureSet"
        assert len(ages) >= len(pts)                       # the reference's ages/points skew is reproduced
        assert got["n_valid"] > 50 and got["n_inliers"] > 20
    # NB on this dense texture ages never exceed 1: the reference's one-slot buckets keep the LAST admitted
    # feature and fresh FAST corners are appended after the tracked ones, so they overwrite them
    # (SURVEY.md row A4) -- reproduced, as the equality with fs.ages above shows.
    assert ages.max() >= 1
    assert np.linalg.norm(frame_pose[:3, 3]) > 0.1 * (nf - 1) * np.linalg.norm(STEP_T)   # the pose actually advanced

    if nf >= 20:
        # row N4: the KITTI segment metric (short segments: this synthetic drive is ~4 m long) of the GPU trajectory
        # against the reference path's is zero to round-off -- parity-level differences do not move it
        from visual_odom_b200 import capi
        seg, t_err, r_err = capi.eval_segments(traj_ref, traj_gpu, lengths=[1.0, 2.0, 3.0], step=2)
        assert len(seg) >= 10 and t_err < 1e-6 and r_err < 1e-5


def test_pipelined_submit_wait_equals_push(ctx):
    """vo_seq_submit / vo_seq_wait with two frames in flight: identical records, point lists, pose and carried state
    to the synchronous vo_seq_push, for gray and for colour input."""
    w, h, nf = 1241, 376, 9
    base, frames = _frames(w, h, 7, nf)
    ctx.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    ref = [ctx.seq_push(l, r) for l, r in frames[1:]]
    pose_ref = ctx.seq_pose()
    state_ref = ctx.seq_state()

    def check(got, k):
        for key in ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters"):
            assert got[key] == ref[k][key], (k, key)
        for key in ("l0", "r0", "l1", "r1", "R", "tvec", "rvec"):
            assert np.array_equal(got[key], ref[k][key]), (k, key)

    ctx.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    ctx.seq_submit(frames[1][0], frames[1][1])
    for k in range(1, nf):
        if k + 1 < nf:
            ctx.seq_submit(frames[k + 1][0], frames[k + 1][1])
            if k == 1:
                with pytest.raises(RuntimeError, match="in flight"):
                    ctx.seq_submit(frames[k + 1][0], frames[k + 1][1])        # a third frame is refused
        check(ctx.seq_wait(), k - 1)
    with pytest.raises(RuntimeError, match="no frame in flight"):
        ctx.seq_wait()
    assert np.array_equal(ctx.seq_pose(), pose_ref)
    st = ctx.seq_state()
    assert all(np.array_equal(a, b) for a, b in zip(st, state_ref))
    # mixing: a synchronous push while a frame is in flight is refused, then works after the wait
    ctx.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    ctx.seq_submit(frames[1][0], frames[1][1])
    with pytest.raises(RuntimeError, match="in flight"):
        ctx.seq_push(frames[2][0], frames[2][1])
    check(ctx.seq_wait(), 0)
    check(ctx.seq_push(frames[2][0], frames[2][1]), 1)


def test_new_calibration_on_a_used_context_equals_a_fresh_context(built):
    """The frame graphs carry the projection matrices in their kernel arguments: a second sequence (and a batch) on the
    SAME context with the same image size but another calibration must not replay the old matrices."""
    from visual_odom_b200.capi import Context
    w, h, nf = 640, 240, 4
    base, frames = _frames(w, h, 13, nf)
    P_l2, P_r2 = base["P_l"].copy(), base["P_r"].copy()
    P_l2[0, 0] *= 1.07; P_l2[1, 1] *= 1.07; P_r2[0, 0] *= 1.07; P_r2[1, 1] *= 1.07; P_r2[0, 3] *= 1.2     # focal length / baseline

    def run(c, P_l, P_r):
        c.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
        return [c.seq_push(l, r) for l, r in frames[1:]]

    used = Context(0, max_features=2048)
    first = run(used, base["P_l"], base["P_r"])           # captures the graphs with the first calibration
    second = run(used, P_l2, P_r2)
    fresh = Context(0, max_features=2048)
    want = run(fresh, P_l2, P_r2)
    for a, b in zip(second, want):
        assert a["n_inliers"] == b["n_inliers"] and np.array_equal(a["tvec"], b["tvec"]) and np.array_equal(a["R"], b["R"])
    assert any(not np.array_equal(a["tvec"], b["tvec"]) for a, b in zip(first, second))      # the calibration matters
    # the batched path caches graphs per unit range too
    u = dict(l0=frames[0][0], r0=frames[0][1], l1=frames[1][0], r1=frames[1][1])
    outs = []
    for c, cals in ((used, [(base["P_l"], base["P_r"]), (P_l2, P_r2)]), (fresh, [(P_l2, P_r2)])):
        for P_l, P_r in cals:
            c.batch_configure(w, h, 1, P_l, P_r)
            arr, keep, pitch = c.make_units([dict(u, n_select=300, t_prev=(0.0, 0.0, -0.2))])
            outs.append(c.frame_batch(arr, pitch)[0])
    assert np.array_equal(outs[1]["tvec"], outs[2]["tvec"]) and outs[1]["n_inliers"] == outs[2]["n_inliers"]
    assert not np.array_equal(outs[0]["tvec"], outs[1]["tvec"])
    used.close(); fresh.close()


def test_host_buffer_calls_do_not_corrupt_a_sequence(built):
    """Entry points that reuse the sequence's image planes are refused while a frame is in flight, and end an idle
    sequence instead of silently corrupting it."""
    from visual_odom_b200.capi import Context
    w, h = 640, 240
    base, frames = _frames(w, h, 17, 4)
    c = Context(0, max_features=2048)
    c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    c.seq_submit(frames[1][0], frames[1][1])
    pts = np.array([[100.5, 80.25], [300.0, 120.0]], np.float32)
    with pytest.raises(RuntimeError, match="have not been waited for"):
        c.lk_track(frames[0][0], frames[1][0], pts)
    with pytest.raises(RuntimeError, match="have not been waited for"):
        c.fast_detect(frames[0][0])
    r1 = c.seq_wait()
    assert r1["n_valid"] > 20
    c.lk_track(frames[0][0], frames[1][0], pts)           # idle sequence: allowed, and the sequence is over
    with pytest.raises(RuntimeError):
        c.seq_push(frames[2][0], frames[2][1])
    c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])      # a new sequence works as before
    r1b = c.seq_push(frames[1][0], frames[1][1])
    assert r1b["n_inliers"] == r1["n_inliers"] and np.array_equal(r1b["tvec"], r1["tvec"])
    c.close()
