"""trackingFrame2Frame(mono_rotation = true) inside the streaming sequence mode (option "mono_rotation", vo_seq_wait_mono).

The reference's header default (src/visualOdometry.h:42) takes `rotation` from findEssentialMat + recoverPose on
pointsLeft_t0 / pointsLeft_t1 (src/visualOdometry.cpp:146-157) and only `translation` from the PnP (:186-189).  The
oracle is the verbatim glue of oracle/ref_path.py with that branch added through cv2 (_mono_ref below), on the synthetic
drive of test_gpu_seq.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

from visual_odom_b200 import synth

STEP_R = np.array([0.001, -0.004, 0.0005])
STEP_T = np.array([0.01, -0.003, -0.2])
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frames(w, h, seed, n):
    base = synth.stereo_unit(w, h, seed)
    out = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=STEP_R * k, tvec=STEP_T * k)
        out.append((u["l1"], u["r1"]))
    return base, out


def _mono_ref(P_l, pL0, pL1):
    """visualOdometry.cpp:146-157 through cv2: focal / pp are the float entries of P_l widened to double.  None where
    cv::findEssentialMat or cv::recoverPose throws (n < 5, no model, a stack of five-point candidates)."""
    import cv2
    focal = float(P_l[0, 0]); pp = (float(P_l[0, 2]), float(P_l[1, 2]))
    try:
        E, mask = cv2.findEssentialMat(pL0, pL1, focal, pp, cv2.RANSAC, 0.999, 1.0)
        n_good, R, t, _ = cv2.recoverPose(E, pL0, pL1, focal=focal, pp=pp, mask=mask.copy())
    except cv2.error:
        return None
    return dict(R=R, t=t.ravel(), mask=mask.ravel().astype(bool), n_good=int(n_good))


def _reference(base, frames, rotation=None):
    """The reference main loop with mono_rotation = true, frame by frame: (pL0, pR0, pL1, pR1, info, mono or None,
    translation, frame_pose, carried FeatureSet).  Where the reference would abort the frame is not integrated and the
    translation carried as the library does (the PnP with < 4 points leaves it untouched).  rotation(pL0, pL1) -> R
    gives the rotation frame_pose integrates (default: cv2's recoverPose)."""
    from oracle import ref_path
    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    out = []
    for k in range(1, len(frames)):
        (l0, r0), (l1, r1) = frames[k - 1], frames[k]
        pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend="cv2")
        mono = _mono_ref(base["P_l"], pL0, pL1)
        if len(pL0) >= 4:
            X = ref_path.triangulate(base["P_l"], base["P_r"], pL0, pR0, "cv2")
            _, translation, _, _ = ref_path.tracking_frame2frame(base["P_l"], pL0, pL1, X, translation, "cv2")
            if mono is not None:
                R = mono["R"] if rotation is None else rotation(pL0, pL1)
                frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
        out.append(dict(pts=(pL0, pR0, pL1, pR1), info=info, mono=mono, t=np.array(translation), pose=frame_pose.copy(),
                        fs=(fs.points.copy(), fs.ages.copy())))
    return out


def _run(c, base, frames, mono, bgr=False):
    """One sequence on context c; returns per-frame (record, pose, state)."""
    c.set_option("mono_rotation", 1 if mono else 0)
    if bgr:
        c.seq_begin_bgr(np.dstack([frames[0][0]] * 3), np.dstack([frames[0][1]] * 3), base["P_l"], base["P_r"])
    else:
        c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    out = []
    for l, r in frames[1:]:
        if bgr:
            c.seq_submit(np.dstack([l] * 3), np.dstack([r] * 3))
            got = c.seq_wait(mono=mono)
        else:
            got = c.seq_push(l, r, mono=mono)
        out.append((got, c.seq_pose(), c.seq_state()))
    return out


PNP_KEYS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")


def _same_record(a, b, mono=True):
    for key in PNP_KEYS:
        assert a[key] == b[key], key
    for key in ("l0", "r0", "l1", "r1", "R", "tvec", "rvec"):
        assert np.array_equal(a[key], b[key]), key
    if mono:
        ma, mb = a["mono"], b["mono"]
        assert all(ma[k] == mb[k] for k in ("status", "n_inliers", "ransac_iters", "n_good"))
        assert np.array_equal(ma["R"], mb["R"]) and np.array_equal(ma["t"], mb["t"])
        assert np.array_equal(a["ess_mask"], b["ess_mask"])


def _stage(c, P_l):
    """vo_mono_rotation (the stage call pinned to cv2 by test_gpu_stages.py) on a frame's point lists: (R, mask, iters)
    or None where it refuses."""
    from visual_odom_b200.capi import VoError
    focal = float(P_l[0, 0]); pp = (float(P_l[0, 2]), float(P_l[1, 2]))

    def run(pL0, pL1):
        try:
            return c.mono_rotation(pL0, pL1, focal, pp)
        except VoError:
            return None
    return run


def _check_against_reference(got_seq, ref, stage, off_seq=None, abort_frames=()):
    """Per frame: point lists and counts bit-exact against the glue; the branch bit-identical to vo_mono_rotation on the
    same lists; against cv2, the rotation within 2e-3 relative.  The five-point solver is not OpenCV's operation for
    operation (INTEGRATION.md section 4).  This drive moves 0.2 m between frames, so most points lie beyond recoverPose's
    distance threshold (50 baselines) and the cheirality vote rests on a few points: there the mask can differ (RANSAC
    stops on another model), and n_good and R can differ at the 1e-4 level even with the same mask.  Returns (max relative R
    difference, frames with another mask than cv2's, frames with another n_good)."""
    worst, differ, good_differ = 0.0, [], []
    for k, ((got, pose, (pts, ages, _)), r) in enumerate(zip(got_seq, ref), start=1):
        pL0, pR0, pL1, pR1 = r["pts"]
        assert got["n_features"] == len(r["info"]["bucketed"]) and got["n_tracked"] == len(r["info"]["kept_idx"]), k
        assert got["n_valid"] == len(pL0), k
        for name, want in zip(("l0", "r0", "l1", "r1"), r["pts"]):
            assert np.array_equal(got[name], want), f"frame {k}: {name}"
        m = got["mono"]
        st = stage(pL0, pL1)
        if r["mono"] is None:
            assert st is None and m["status"] != 0 and np.array_equal(got["R"], np.eye(3)), f"frame {k}: the reference aborts here"
        else:
            assert m["status"] == 0 and st is not None, k
            Rs, ms, its = st
            assert np.array_equal(got["ess_mask"], ms) and np.array_equal(m["R"], Rs), f"frame {k}: sequence != vo_mono_rotation"
            assert m["n_inliers"] == int(ms.sum()) and m["ransac_iters"] == its, k
            assert np.array_equal(got["R"], m["R"]), k                   # the record's R is the mono rotation
            rel = np.linalg.norm(m["R"] - r["mono"]["R"]) / np.linalg.norm(r["mono"]["R"])
            worst = max(worst, rel)
            assert rel <= 2e-3, f"frame {k}: rotation off cv2's by {rel:.2e}"
            if not np.array_equal(got["ess_mask"], r["mono"]["mask"]):
                differ.append(k)
            if m["n_good"] != r["mono"]["n_good"]:
                good_differ.append(k)
        assert k not in abort_frames or r["mono"] is None, k
        assert np.abs(pose - r["pose"]).max() <= 1e-6 * max(1.0, np.abs(r["pose"]).max()), f"frame {k}: frame_pose"
        assert np.array_equal(pts, r["fs"][0]) and np.array_equal(ages, r["fs"][1]), f"frame {k}: carried FeatureSet"
        if off_seq is not None:                     # the PnP's values are the same bits as without the branch
            off = off_seq[k - 1][0]
            for key in ("tvec", "rvec"):
                assert np.array_equal(got[key], off[key]), (k, key)
            assert got["n_inliers"] == off["n_inliers"] and got["ransac_iters"] == off["ransac_iters"], k
            assert got["pnp_status"] == off["pnp_status"], k
    return worst, differ, good_differ


# ----------------------------------------------------------------------------------------------------- CPU (no GPU)
def test_mono_oracle_recovers_the_drive_rotation():
    """The test's oracle is itself sound: on the synthetic drive (frame k rendered at Rodrigues(k STEP_R) about one axis, so
    consecutive frames differ by exactly Rodrigues(STEP_R), a 4.2e-3 rad turn) cv2's findEssentialMat + recoverPose, fed
    the point lists the reference glue produces, recovers that rotation.  Tolerance 1.5e-3 rad: with ~230 matches and a
    0.2 m baseline the five-point estimate trades rotation against translation by a few 1e-4 rad (6.4e-4 at most over
    these frames), while a transposed or otherwise wrong convention is off by twice the turn (8e-3 rad)."""
    cv2 = pytest.importorskip("cv2")
    base, frames = _frames(1241, 376, 31, 8)
    ref = _reference(base, frames)
    R_step, _ = cv2.Rodrigues(STEP_R.reshape(3, 1))
    for k, r in enumerate(ref, start=1):
        assert r["mono"] is not None, k
        err = np.linalg.norm(cv2.Rodrigues(r["mono"]["R"] @ R_step.T)[0])
        assert err <= 1.5e-3, f"frame {k}: {err:.2e} rad from the rendered rotation"
        assert np.linalg.norm(cv2.Rodrigues(r["mono"]["R"] @ R_step)[0]) > 5e-3
        assert r["mono"]["mask"].sum() > 0.9 * len(r["pts"][0])


def test_run_sequence_check_accepts_mono_rotation(built, tmp_path):
    cv2 = pytest.importorskip("cv2")
    for cam in ("image_0", "image_1"):
        (tmp_path / cam).mkdir()
        for i in range(2):
            cv2.imwrite(str(tmp_path / cam / ("%06d.png" % i)), np.full((40, 64), 100 + i, np.uint8))
    cal = tmp_path / "cal.yaml"
    cal.write_text("Camera.fx: 718.856\nCamera.fy: 718.856\nCamera.cx: 607.1928\nCamera.cy: 185.2157\nCamera.bf: -386.1448\n")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_sequence.py"), str(tmp_path) + "/", str(cal),
                        "--check", "--mono-rotation"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    assert "2 stereo pairs of 64x40" in r.stdout and "recoverPose" in r.stdout


# ----------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("w,h,nf", [(1241, 376, 22), (640, 480, 6)])
def test_mono_sequence_matches_reference(built, w, h, nf):
    pytest.importorskip("cv2")
    from visual_odom_b200.capi import Context
    base, frames = _frames(w, h, 31, nf)
    st_ctx = Context(0, max_features=4096)
    stage = _stage(st_ctx, base["P_l"])
    ref = _reference(base, frames, rotation=lambda a, b: stage(a, b)[0])
    off_ctx = Context(0, max_features=4096)
    off = _run(off_ctx, base, frames, mono=False)
    off_ctx.close()
    c = Context(0, max_features=4096)
    got = _run(c, base, frames, mono=True)
    worst, differ, good_differ = _check_against_reference(got, ref, stage, off_seq=off)
    print(f"{w}x{h}, {nf - 1} frames: max relative difference of R from cv2's recoverPose {worst:.2e}; frames with another "
          f"essential mask than cv2: {differ}; with another n_good: {good_differ}")
    st_ctx.close()
    assert all(g[0]["n_valid"] > 50 for g in got)
    # plain vo_seq_wait on a mono sequence: the same record (R = the mono rotation), only the details are missing
    c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    plain = [c.seq_push(l, r) for l, r in frames[1:]]
    for a, (b, _, _) in zip(plain, got):
        _same_record(a, b, mono=False)
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("graphs", [1, 0])
def test_mono_pipelined_equals_push(built, graphs):
    """vo_seq_submit / vo_seq_wait_mono with two frames in flight: records, mono results, masks, pose and state identical
    to the synchronous push, for gray and BGR input, with and without CUDA graphs."""
    from visual_odom_b200.capi import Context
    base, frames = _frames(1241, 376, 7, 9)
    c = Context(0, max_features=4096)
    c.set_option("graphs", graphs)
    want = _run(c, base, frames, mono=True)
    for bgr in (False, True):
        c.set_option("mono_rotation", 1)
        if bgr:
            c.seq_begin_bgr(np.dstack([frames[0][0]] * 3), np.dstack([frames[0][1]] * 3), base["P_l"], base["P_r"])
            sub = [(np.dstack([l] * 3), np.dstack([r] * 3)) for l, r in frames[1:]]
        else:
            c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
            sub = frames[1:]
        c.seq_submit(*sub[0])
        for k in range(len(sub)):
            if k + 1 < len(sub):
                c.seq_submit(*sub[k + 1])
            _same_record(c.seq_wait(mono=True), want[k][0])
        assert np.array_equal(c.seq_pose(), want[-1][1])
        assert all(np.array_equal(a, b) for a, b in zip(c.seq_state(), want[-1][2]))
    c.close()


@pytest.mark.gpu
def test_mono_abort_frame_is_reported_and_skipped(built):
    """A pair whose right image is uniform leaves fewer than 5 valid matches: cv::findEssentialMat would throw.  The frame
    reports VO_E_TOO_FEW_POINTS with R = I, frame_pose does not move, and the frames after it match the reference glue
    again, carried state included."""
    pytest.importorskip("cv2")
    from visual_odom_b200.capi import Context, VO_E_TOO_FEW_POINTS
    base, frames = _frames(1241, 376, 31, 12)
    j = 6
    frames[j] = (frames[j][0], np.full_like(frames[j][1], 128))
    st_ctx = Context(0, max_features=4096)
    stage = _stage(st_ctx, base["P_l"])
    ref = _reference(base, frames, rotation=lambda a, b: stage(a, b)[0])
    c = Context(0, max_features=4096)
    got = _run(c, base, frames, mono=True)
    _check_against_reference(got, ref, stage, abort_frames=(j,))
    st_ctx.close()
    rec, pose, _ = got[j - 1]
    assert rec["n_valid"] < 5 and rec["mono"]["status"] == VO_E_TOO_FEW_POINTS and np.array_equal(rec["R"], np.eye(3))
    assert np.array_equal(pose, got[j - 2][1])
    assert all(g[0]["mono"]["status"] == 0 for g in got[j + 1:])       # the sequence recovers
    c.close()


@pytest.mark.gpu
def test_mono_mode_switches_on_one_context(built):
    """off -> on -> off on one context: each sequence equals a fresh context in that mode; vo_seq_wait_mono is refused
    on a mono-off sequence; vo_mono_rotation between frames of an idle mono sequence matches cv2 and leaves the sequence's
    results unchanged."""
    cv2 = pytest.importorskip("cv2")
    from visual_odom_b200.capi import Context
    base, frames = _frames(1241, 376, 13, 6)
    fresh = {}
    for mono in (False, True):
        f = Context(0, max_features=4096)
        fresh[mono] = _run(f, base, frames, mono=mono)
        f.close()
    c = Context(0, max_features=4096)
    for mono in (False, True, False):
        got = _run(c, base, frames, mono=mono)
        for (a, pa, _), (b, pb, _) in zip(got, fresh[mono]):
            _same_record(a, b, mono=mono)
            assert np.array_equal(pa, pb)
    c.set_option("mono_rotation", 0)
    c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    c.seq_submit(*frames[1])
    with pytest.raises(RuntimeError, match="mono_rotation"):
        c.seq_wait(mono=True)
    c.seq_wait()
    # the stage call between two frames of a mono sequence
    c.set_option("mono_rotation", 1)
    c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
    first = [c.seq_push(l, r, mono=True) for l, r in frames[1:3]]
    p0, p1, focal, pp = synth.essential_stress_set(1500, 0.15, 0.3, 5)
    E, mask = cv2.findEssentialMat(p0, p1, focal, pp, cv2.RANSAC, 0.999, 1.0)
    _, R, _, _ = cv2.recoverPose(E, p0, p1, focal=focal, pp=pp, mask=mask.copy())
    Rg, mg, _ = c.mono_rotation(p0, p1, focal, pp)
    assert np.array_equal(mg, mask.ravel().astype(bool)) and np.linalg.norm(Rg - R) <= 1e-6 * np.linalg.norm(R)
    rest = [c.seq_push(l, r, mono=True) for l, r in frames[3:]]
    for a, (b, _, _) in zip(first + rest, fresh[True]):
        _same_record(a, b)
    assert np.array_equal(c.seq_pose(), fresh[True][-1][1])
    c.close()
