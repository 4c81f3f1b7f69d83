"""The sequence modes' feature bookkeeping on long-lived tracks, against the reference path.

synth.blob_sequence is a sparse drive on which features live for 10+ frames (tests/test_oracle_long_tracks.py checks that
it does): the age gate of Bucket::add_feature refuses features aged 10 or more, refills pair fresh corners with stale
ages (the ages keep their pre-check length while the points shrink) and frames run with a handful of matches.  Here the
GPU glue kernels (k_seq_append / k_seq_bucket / k_seq_carry of csrc/seq.cu) in vo_seq_* and vo_mseq_*, and the host glue
of the C++ facade, are held to the cv2 reference path on that drive frame by frame, carried ages included."""
import os
import struct
import subprocess

import numpy as np
import pytest

from visual_odom_b200 import synth
from test_oracle_long_tracks import reference_run, scene_edges

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COUNTS = ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters", "pnp_status")
ARRAYS = ("rvec", "tvec", "R", "l0", "r0", "l1", "r1")
# the second blob drive (multi-sequence and facade tests): another seed and another soft stretch (frames 5..19), so the
# gate refuses features on other frames than in the first
OTHER = dict(seed=6, sharp=lambda k: k < 5 or k >= 20)


@pytest.fixture(scope="module")
def blobs():
    return synth.blob_sequence()


@pytest.fixture(scope="module")
def reference(blobs):
    P_l, P_r, frames = blobs
    return reference_run(P_l, P_r, frames)


@pytest.fixture(scope="module")
def other():
    return synth.blob_sequence(**OTHER)


@pytest.fixture(scope="module")
def other_reference(other):
    P_l, P_r, frames = other
    return reference_run(P_l, P_r, frames, spy=True)


def _push_all(c, P_l, P_r, frames, mono=False):
    """One sequence through vo_seq_push: per frame (record, frame_pose, carried state)."""
    c.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    out = []
    for l, r in frames[1:]:
        got = c.seq_push(l, r, mono=mono)
        out.append((got, c.seq_pose(), c.seq_state()))
    return out


@pytest.fixture(scope="module")
def pushed(ctx, blobs):
    P_l, P_r, frames = blobs
    return _push_all(ctx, P_l, P_r, frames)


def _check_against_reference(got_seq, ref):
    """Per frame: counts and pnp_status, the four point lists and the carried points AND ages bit for bit; R and t within
    1e-4 of cv2, frame_pose within 1e-6."""
    for k, ((got, pose, (pts, ages, _)), r) in enumerate(zip(got_seq, ref), start=1):
        pL0 = r["pts"][0]
        assert got["n_features"] == len(r["info"]["bucketed"]), f"frame {k}: bucketed feature count"
        assert got["n_tracked"] == len(r["info"]["kept_idx"]), f"frame {k}: circular-check survivors"
        assert got["n_valid"] == len(pL0), f"frame {k}: valid matches"
        assert got["pnp_status"] == r["pnp_status"], f"frame {k}: pnp_status"
        assert got["n_inliers"] == len(r["inliers"]), f"frame {k}: inlier count"
        for name, want in zip(("l0", "r0", "l1", "r1"), r["pts"]):
            assert np.array_equal(got[name], want), f"frame {k}: {name}"
        assert np.array_equal(pts, r["fs"][0]), f"frame {k}: carried points"
        assert np.array_equal(ages, r["fs"][1]), f"frame {k}: carried ages"
        if r["R"] is not None:
            assert np.linalg.norm(got["R"] - r["R"]) / np.linalg.norm(r["R"]) <= 1e-4, f"frame {k}: R"
        assert np.linalg.norm(got["tvec"] - r["t"]) / np.linalg.norm(r["t"]) <= 1e-4, f"frame {k}: t"
        assert np.abs(pose - r["pose"]).max() <= 1e-6 * max(1.0, np.abs(r["pose"]).max()), f"frame {k}: frame_pose"


def _same_record(a, b, where):
    for key in COUNTS:
        assert a[key] == b[key], f"{where}: {key} {a[key]} != {b[key]}"
    for key in ARRAYS:
        assert a[key].dtype == b[key].dtype and np.array_equal(a[key], b[key]), f"{where}: {key}"


def _same_state(a, b, where):
    for name, x, y in zip(("points", "ages", "translation"), a, b):
        assert x.dtype == y.dtype and np.array_equal(x, y), f"{where}: carried {name}"


def test_seq_push_matches_reference_on_long_tracks(pushed, reference):
    _check_against_reference(pushed, reference)
    # the drive reached the gate on the GPU side too: some carried feature aged 10 entered a frame's bucketing
    assert any((ages[:len(pts)] >= 10).any() for _, _, (pts, ages, _) in pushed)
    assert min(g["n_valid"] for g, _, _ in pushed) < 10


def test_pipelined_submit_wait_equals_push(ctx, blobs, pushed):
    """Two frames in flight: records, point lists, carried state and frame_pose identical to vo_seq_push."""
    P_l, P_r, frames = blobs
    ctx.seq_begin(frames[0][0], frames[0][1], P_l, P_r)
    ctx.seq_submit(*frames[1])
    for k in range(1, len(frames)):
        if k + 1 < len(frames):
            ctx.seq_submit(*frames[k + 1])
        got = ctx.seq_wait()
        _same_record(got, pushed[k - 1][0], f"frame {k}")
    assert np.array_equal(ctx.seq_pose(), pushed[-1][1])
    _same_state(ctx.seq_state(), pushed[-1][2], "last frame")


def _dense_drive(n):
    base = synth.stereo_unit(1241, 376, 31)
    out = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(1241, 376, 31, rvec=synth.SEQ_STEP_R * k, tvec=synth.SEQ_STEP_T * k)
        out.append((u["l1"], u["r1"]))
    return out


def test_mseq_diverging_counts_match_running_alone(ctx, blobs, other, reference, pushed):
    """Three sequences in lockstep at 1241x376: two blob drives whose gates fire on different frames and one dense drive.
    The per-sequence strides of the glue kernels see very different counts; each sequence must be bit-identical to
    running it alone, and blob sequence 0 must match the reference path."""
    from visual_odom_b200 import capi
    P_l, P_r, frames0 = blobs
    frames1 = other[2]
    seqs = [frames0, frames1, _dense_drive(len(frames0))]
    n = len(seqs)
    ctx.mseq_begin([s[0][0] for s in seqs], [s[0][1] for s in seqs], P_l, P_r)
    run = []
    for k in range(1, len(frames0)):
        ctx.mseq_submit([s[k][0] for s in seqs], [s[k][1] for s in seqs])
        recs = ctx.mseq_wait()
        run.append([(recs[q], ctx.mseq_pose(q), ctx.mseq_state(q)) for q in range(n)])
    for q in range(n):
        alone = pushed if q == 0 else _push_all(ctx, P_l, P_r, seqs[q])
        for k, (per_q, (a, pose, st)) in enumerate(zip(run, alone), start=1):
            rec, mpose, mst = per_q[q]
            assert rec["status"] == capi.VO_OK
            _same_record(rec, a, f"sequence {q} frame {k}")
            _same_state(mst, st, f"sequence {q} frame {k}")
            assert np.array_equal(mpose, pose), f"sequence {q} frame {k}: frame_pose"
    _check_against_reference([per_q[0] for per_q in run], reference)

    def gate_frames(q):        # frames whose carried state pairs a point with an age >= 10 (next frame's bucketing)
        return {k for k, per_q in enumerate(run, start=1) if (per_q[q][2][1][:len(per_q[q][2][0])] >= 10).any()}
    g0, g1 = gate_frames(0), gate_frames(1)
    assert g0 and g1 and g0 != g1 and not gate_frames(2)
    counts = [[per_q[q][0]["n_features"] for per_q in run] for q in range(n)]
    assert any(len({c[k] for c in counts}) == n for k in range(len(run)))        # the counts do diverge


def _facade_run(tmp_path, P_l, P_r, frames):
    w, h, nf = frames[0][0].shape[1], frames[0][0].shape[0], len(frames)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("<iii", w, h, nf))
        f.write(P_l.astype(np.float32).tobytes()); f.write(P_r.astype(np.float32).tobytes())
        for l, r in frames:
            f.write(l.tobytes()); f.write(r.tobytes())
    r = subprocess.run([os.path.join(ROOT, "tests", "cpp", "facade_main"), fin, fout], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    return open(fout, "rb").read()


def test_facade_matches_reference_on_long_tracks(built, ctx, tmp_path, other, other_reference):
    """tests/cpp/facade_main (the reference's main loop over the C++ facade) on the second blob drive, whose gate refuses
    features aged exactly 10 on frames 14 and 15: point lists, triangulated points, inliers, R / t, the FeatureSet size
    and frame_pose against the reference path.

    facade_main also runs the mono_rotation branch on every frame.  On this drive cv2.findEssentialMat returns one 3x3 E
    on every frame (asserted), so the facade never takes its refusal path (it throws from vo_mono_rotation where the
    reference aborts; the five-match refusal is pinned on vo_mono_rotation itself in test_gpu_pnp_edges.py and in the
    sequence mode below).  The facade's rotation must be vo_mono_rotation's on the same lists bit for bit (that stage is
    pinned to cv2 in test_gpu_stages.py), and the flag must not change the translation.  Its value is not compared with
    cv2's: with 6-40 matches 10-45 m away and a 0.2 m step, every five-point model fits nearly all matches within
    RANSAC's 1 px, the cheirality vote is weak, and cv2 itself returns the twisted-pair rotation (pi off the rendered
    step) on some frames of these drives."""
    import cv2
    P_l, P_r, frames = other
    assert any(age == 10 for _, age in scene_edges(other_reference)["gated"])     # `age <= 10` would differ here
    buf = _facade_run(tmp_path, P_l, P_r, frames)
    off = 0

    def take(dtype, count):
        nonlocal off
        a = np.frombuffer(buf, dtype, count, off)
        off += a.nbytes
        return a

    focal = float(P_l[0, 0]); pp = (float(P_l[0, 2]), float(P_l[1, 2]))
    for k, r in enumerate(other_reference, start=1):
        pL0, pR0, pL1, pR1 = r["pts"]
        n = int(take(np.int32, 1)[0])
        assert n == len(pL0), f"frame {k}: {n} vs {len(pL0)} matched features"
        for name, want in zip(("l0", "r0", "l1", "r1"), r["pts"]):
            assert np.array_equal(take(np.float32, 2 * n).reshape(-1, 2), want), f"frame {k}: {name}"
        assert np.array_equal(take(np.float32, 3 * n).reshape(-1, 3), r["X"]), f"frame {k}: X"
        ni = int(take(np.int32, 1)[0])
        assert np.array_equal(take(np.int32, ni), r["inliers"]), f"frame {k}: inlier list"
        Rg = take(np.float64, 9).reshape(3, 3); tg = take(np.float64, 3)
        assert np.linalg.norm(Rg - r["R"]) / np.linalg.norm(r["R"]) <= 1e-4, f"frame {k}: R"
        assert np.linalg.norm(tg - r["t"]) / np.linalg.norm(r["t"]) <= 1e-4, f"frame {k}: t"
        assert int(take(np.int32, 1)[0]) == len(r["fs"][0]), f"frame {k}: fs.size()"
        pose_g = take(np.float64, 16).reshape(4, 4)
        assert np.abs(pose_g - r["pose"]).max() <= 1e-6 * max(1.0, np.abs(r["pose"]).max()), f"frame {k}: frame_pose"
        take(np.float32, 4 * n)                              # Frame::triangulateFeaturePoints (test_gpu_facade.py)
        Rm_g = take(np.float64, 9).reshape(3, 3); tm_g = take(np.float64, 3)
        E, _ = cv2.findEssentialMat(pL0, pL1, focal, pp, cv2.RANSAC, 0.999, 1.0)
        assert E is not None and E.shape == (3, 3), f"frame {k}: cv::recoverPose would throw on this drive"
        assert np.array_equal(Rm_g, ctx.mono_rotation(pL0, pL1, focal, pp)[0]), f"frame {k}: mono rotation"
        assert np.array_equal(tm_g, tg), f"frame {k}: the PnP translation does not depend on the flag"
    assert off == len(buf)


def test_mono_rotation_leaves_the_pnp_and_the_state_alone(built, ctx, blobs, pushed):
    """The option mono_rotation on, over the blob drive: every PnP field and the carried state are those of the
    option-off run; where the branch succeeds, R is vo_mono_rotation on that frame's lists; where it refuses, R = I."""
    from visual_odom_b200.capi import Context, VoError, VO_E_TOO_FEW_POINTS
    P_l, P_r, frames = blobs
    c = Context(0, max_features=4096)
    c.set_option("mono_rotation", 1)
    got = _push_all(c, P_l, P_r, frames, mono=True)
    c.close()
    focal = float(P_l[0, 0]); pp = (float(P_l[0, 2]), float(P_l[1, 2]))
    refused = 0
    pose_exp = np.eye(4)
    for k, ((a, pose, st), (b, _, st_off)) in enumerate(zip(got, pushed), start=1):
        for key in COUNTS:
            assert a[key] == b[key], f"frame {k}: {key}"
        for key in ("tvec", "rvec", "l0", "r0", "l1", "r1"):
            assert np.array_equal(a[key], b[key]), f"frame {k}: {key}"
        _same_state(st, st_off, f"frame {k}")
        if a["mono"]["status"] == 0:
            Rs, ms, its = ctx.mono_rotation(a["l0"], a["l1"], focal, pp)
            assert np.array_equal(a["R"], Rs) and np.array_equal(a["ess_mask"], ms), f"frame {k}: R != vo_mono_rotation"
            assert a["mono"]["ransac_iters"] == its, f"frame {k}"
            from oracle import ref_path
            pose_exp = ref_path.integrate_pose(pose_exp, a["R"], a["tvec"])
        else:
            assert a["mono"]["status"] == VO_E_TOO_FEW_POINTS and np.array_equal(a["R"], np.eye(3)), f"frame {k}"
            with pytest.raises(VoError):
                ctx.mono_rotation(a["l0"], a["l1"], focal, pp)
            refused += 1
        assert np.abs(pose - pose_exp).max() <= 1e-9 * max(1.0, np.abs(pose_exp).max()), f"frame {k}: frame_pose"
    assert refused > 0 and refused < len(got)
