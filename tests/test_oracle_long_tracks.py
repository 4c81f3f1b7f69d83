"""The feature bookkeeping of the reference's main loop on long-lived tracks, CPU side.

On the dense textures of the other sequence tests every frame appends fresh FAST corners into every bucket after the
tracked features, the last admitted feature wins the cell, and ages never pass 1.  So neither the age gate of
Bucket::add_feature (a feature aged 10 or more is refused) nor the ages / points length skew after the circular check
ever decides anything there.  synth.blob_sequence renders a sparse drive whose features live for 10+ frames; this file
checks that the scene really reaches those rules through the cv2 reference path, that the C oracle agrees with cv2 on it,
and pins the gate on a hand-built FeatureSet.  tests/test_gpu_long_tracks.py holds the GPU kernels and the facade to the
same reference on the same scene."""
import numpy as np
import pytest

from visual_odom_b200 import synth

cv2 = pytest.importorskip("cv2")

STEP_T = synth.SEQ_STEP_T
VO_OK, VO_PNP_NO_MODEL, VO_E_TOO_FEW_POINTS = 0, 1, -3          # include/vo_b200.h


def reference_run(P_l, P_r, frames, backend="cv2", spy=False):
    """The reference main loop (oracle/ref_path.py glue) frame by frame.  Per frame: the four point lists, info, the
    PnP's R / translation / inliers, the pnp_status the library reports for that outcome, frame_pose and the carried
    FeatureSet.  A frame with < 4 matches keeps the translation and does not move frame_pose (the reference would abort
    in cv::solvePnPRansac).  spy=True also records what bucketing and the refill saw: ("bucket_in", points, ages, rows,
    cols, bucket_size) and ("refill", n_points before, ages before, corners appended, ages after)."""
    from oracle import ref_path
    events = []
    real_bucket, real_append = ref_path.bucketing_features, ref_path.append_new_features

    def bucket(rows, cols, features, bucket_size, per_bucket):
        events.append(("bucket_in", features.points.copy(), features.ages.copy(), rows, cols, bucket_size))
        real_bucket(rows, cols, features, bucket_size, per_bucket)

    def append(img, features, backend="cv2"):
        n_pts, ages = features.size(), features.ages.copy()
        real_append(img, features, backend)
        events.append(("refill", n_pts, ages, features.size() - n_pts, features.ages.copy()))

    fs = ref_path.FeatureSet()
    translation = np.zeros(3)
    frame_pose = np.eye(4)
    out = []
    if spy:
        ref_path.bucketing_features, ref_path.append_new_features = bucket, append
    try:
        for k in range(1, len(frames)):
            (l0, r0), (l1, r1) = frames[k - 1], frames[k]
            del events[:]
            pL0, pR0, pL1, pR1, info = ref_path.matching_features(l0, r0, l1, r1, fs, backend=backend)
            X = ref_path.triangulate(P_l, P_r, pL0, pR0, backend)
            R, inl, status = None, np.zeros(0, np.int32), VO_E_TOO_FEW_POINTS
            if len(pL0) >= 4:
                R, translation, inl, _ = ref_path.tracking_frame2frame(P_l, pL0, pL1, X, translation, backend)
                status = VO_OK if len(inl) else VO_PNP_NO_MODEL
                frame_pose = ref_path.integrate_pose(frame_pose, R, translation)
            out.append(dict(pts=(pL0, pR0, pL1, pR1), info=info, X=X, R=R, t=np.array(translation), inliers=inl,
                            pnp_status=status, pose=frame_pose.copy(), fs=(fs.points.copy(), fs.ages.copy()),
                            events=list(events)))
    finally:
        ref_path.bucketing_features, ref_path.append_new_features = real_bucket, real_append
    return out


def refused_by_the_gate(pts, ages, rows, cols, bucket_size):
    """Indices of the bucketing input that the age gate alone keeps out: aged >= 10 and the last entry of their cell, so
    that without the gate they would have won the one-slot bucket."""
    nw = cols // bucket_size
    cell = (pts[:, 1] / np.float32(bucket_size)).astype(np.int32) * nw + (pts[:, 0] / np.float32(bucket_size)).astype(np.int32)
    last = {c: i for i, c in enumerate(cell)}
    return [i for i in range(len(pts)) if ages[i] >= 10 and last[cell[i]] == i]


def scene_edges(ref):
    """What a run of reference_run(spy=True) reached: (frame, age) of each feature the gate alone refused, refills that
    paired a fresh corner with a stale non-zero age, the largest carried age, frames with 5 <= n_valid < 10, and frames
    with n_valid >= 10 whose translation is off the true 0.2 m by more than 20 %."""
    gated, stale, max_age, few, off = [], [], 0, [], []
    for k, r in enumerate(ref, start=1):
        for ev in r["events"]:
            if ev[0] == "bucket_in":
                _, pts, ages = ev[:3]
                gated += [(k, int(ages[i])) for i in refused_by_the_gate(pts, ages[:len(pts)], *ev[3:])]
            else:
                _, n_pts, ages_before, n_new, ages_after = ev
                if n_new > 0 and len(ages_before) > n_pts and ages_after[n_pts] != 0:
                    stale.append(k)
        if len(r["fs"][1]):
            max_age = max(max_age, int(r["fs"][1].max()))
        n = len(r["pts"][0])
        if 5 <= n < 10:
            few.append(k)
        if n >= 10 and abs(np.linalg.norm(r["t"]) - np.linalg.norm(STEP_T)) > 0.2 * np.linalg.norm(STEP_T):
            off.append(k)
    return dict(gated=gated, stale=stale, max_age=max_age, few=few, off=off)


@pytest.fixture(scope="module")
def blobs():
    return synth.blob_sequence()


@pytest.fixture(scope="module")
def blob_ref(blobs):
    P_l, P_r, frames = blobs
    return reference_run(P_l, P_r, frames, spy=True)


def test_blob_sequence_is_deterministic_and_sparse(blobs):
    P_l, P_r, frames = blobs
    again = synth.blob_sequence()[2]
    assert len(frames) == 24 and all(l.shape == (376, 1241) and l.dtype == np.uint8 for l, _ in frames)
    assert all(np.array_equal(a, c) and np.array_equal(b, d) for (a, b), (c, d) in zip(frames, again))
    assert not np.array_equal(synth.blob_sequence(seed=5, n_frames=2)[2][0][0], frames[0][0])
    assert np.array_equal(P_l, synth.proj_matrices()[0]) and np.array_equal(P_r, synth.proj_matrices()[1])
    # FAST fires on the sharp frames and hardly on the soft ones (only where blobs overlap)
    from oracle import ref_path
    n_sharp, n_soft = len(ref_path.fast_cv2(frames[0][0])), len(ref_path.fast_cv2(frames[10][0]))
    assert n_sharp > 50 and n_soft < n_sharp // 10


def test_blob_scene_reaches_the_age_gate_and_the_skew(blob_ref):
    e = scene_edges(blob_ref)
    # the gate alone refuses features, among them some aged exactly 10 (where `age <= 10` would differ)
    assert e["gated"] and any(a == 10 for _, a in e["gated"]), e["gated"]
    assert e["stale"], "no refill paired a fresh corner with a stale age"
    assert e["max_age"] >= 10
    assert e["few"], "no frame ran with 5..9 valid matches"
    assert not e["off"], f"translation off the drive on frames {e['off']}"
    assert all(len(r["pts"][0]) >= 4 for r in blob_ref)        # every frame reaches the PnP


def test_dense_texture_never_reaches_the_gate():
    """Why the blob scene exists: the dense drive of the other sequence tests refills every bucket on every frame, so no
    age reaches 10 and the gate never refuses a feature."""
    frames = []
    base = synth.stereo_unit(640, 240, 31)
    frames.append((base["l0"], base["r0"]))
    for k in range(1, 12):
        u = synth.stereo_unit(640, 240, 31, rvec=synth.SEQ_STEP_R * k, tvec=STEP_T * k)
        frames.append((u["l1"], u["r1"]))
    e = scene_edges(reference_run(base["P_l"], base["P_r"], frames, spy=True))
    assert not e["gated"] and e["max_age"] < 10 and not e["few"]


def test_c_oracle_matches_cv2_on_the_blob_scene(built, blobs, blob_ref):
    """backend="c" (oracle/lk_ref.c, fast_ref.c, pnp_ref.py) against cv2 on every frame: the point lists, the kept
    indices, the triangulated points, the inliers and the carried FeatureSet bit for bit, the pose to round-off."""
    P_l, P_r, frames = blobs
    got = reference_run(P_l, P_r, frames, backend="c")
    for k, (a, b) in enumerate(zip(got, blob_ref), start=1):
        for name, x, y in zip(("l0", "r0", "l1", "r1"), a["pts"], b["pts"]):
            assert np.array_equal(x, y), f"frame {k}: {name}"
        assert np.array_equal(a["info"]["bucketed"], b["info"]["bucketed"]), f"frame {k}: bucketed"
        assert np.array_equal(a["info"]["kept_idx"], b["info"]["kept_idx"]), f"frame {k}: kept indices"
        assert np.array_equal(a["fs"][0], b["fs"][0]) and np.array_equal(a["fs"][1], b["fs"][1]), f"frame {k}: FeatureSet"
        assert np.array_equal(a["inliers"], b["inliers"]) and a["pnp_status"] == b["pnp_status"], f"frame {k}: inliers"
        assert np.linalg.norm(a["t"] - b["t"]) <= 1e-4 * np.linalg.norm(b["t"]), f"frame {k}: translation"


# 376 x 1241 (the KITTI size): bucket_size = 376 / 10 = 37, nh = 10, nw = 33, (nh + 1) (nw + 1) = 374 buckets addressed
# as h * nw + w.  Input in order: (x, y, age)
GATE_INPUT = [
    (190.0, 80.0, 3),        # cell (2, 5) = 71: admitted
    (200.5, 90.5, 9),        # cell 71: admitted, overwrites the one-slot bucket (the last admitted wins)
    (185.25, 100.0, 10),     # cell 71: refused (age 10)
    (220.0, 110.0, 11),      # cell 71: refused (age 11)
    (500.0, 300.0, 10),      # cell (8, 13) = 277: refused, the cell stays empty
    (1230.5, 160.25, 2),     # cell (4, 33) = 165 = cell (5, 0): admitted
    (10.0, 200.0, 0),        # cell (5, 0) = 165: overwrites the aliased (4, 33) entry
    (1235.0, 50.0, 9),       # cell (1, 33) = 66 = cell (2, 0): admitted
    (5.0, 90.0, 10),         # cell (2, 0) = 66: refused, the aliased entry stays
    (600.0, 372.0, 1),       # cell (10, 16) = 346: the bottom partial row, read back once
]
# read-back order h = 0..10, w = 0..33 of cells h * 33 + w: (1, 33) = 66, (2, 0) = 66, (2, 5) = 71, (4, 33) = 165,
# (5, 0) = 165, (8, 13) = 277 (empty), (10, 16) = 346
GATE_OUTPUT = [((1235.0, 50.0), 9), ((1235.0, 50.0), 9), ((200.5, 90.5), 9), ((10.0, 200.0), 0), ((10.0, 200.0), 0),
               ((600.0, 372.0), 1)]


def test_bucketing_gate_by_hand():
    """bucketingFeatures + Bucket::add_feature (reference src/feature.cpp:206-253, src/bucket.cpp:14-45) on a hand-built
    FeatureSet: ages 9, 10 and 11 in one cell, the last admitted feature winning, and the aliased cells
    (h, nw) = (h + 1, 0) read back twice."""
    from oracle import ref_path
    fs = ref_path.FeatureSet()
    fs.points = np.array([(x, y) for x, y, _ in GATE_INPUT], np.float32)
    fs.ages = np.array([a for _, _, a in GATE_INPUT], np.int32)
    ref_path.bucketing_features(376, 1241, fs, 376 // 10, 1)
    assert np.array_equal(fs.points, np.array([p for p, _ in GATE_OUTPUT], np.float32))
    assert np.array_equal(fs.ages, np.array([a for _, a in GATE_OUTPUT], np.int32))
    # the gate is `age < 10`: at `<= 10` the age-10 entries would win cells 71, 277 and 66
    b = ref_path.Bucket(1)
    for age in (9, 10, 11):
        b.add_feature((float(age), 0.0), age)
    assert b.points == [(9.0, 0.0)] and b.ages == [9]
