"""The sequence modes' bucketing parameters on the CPU: vo_params.refill_threshold, bucket_rows_divisor,
features_per_bucket and bucket_age_threshold (the literals 2000, rows / 10, 1 and 10 of the reference's matchingFeatures()
and Bucket::add_feature).

oracle/ref_path.py restates the reference at its literals.  This file restates Bucket / bucketingFeatures
(src/bucket.cpp, src/feature.cpp:206-253) literally with the age threshold and bucket size as arguments, and
matchingFeatures (src/visualOdometry.cpp:81-129) on top of ref_path's other pieces with the four values as keywords
(matching_features below, which tests/test_gpu_bucketing.py holds the GPU to).  At the literals both equal ref_path's; at
every value the literal bucketing equals the closed form k_seq_bucket (csrc/seq.cu) computes: a cell whose admitted
features are a_1 .. a_c in input order reads back as a_1 .. a_c when c <= k and as a_c, a_2, .. a_k when c > k.  The
vo_params struct is held to the header's layout."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from visual_odom_b200 import capi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_FIELDS = dict(refill_threshold=2000, bucket_rows_divisor=10, features_per_bucket=1, bucket_age_threshold=10)


# ----------------------------------------------------------------------------- literal transcription of the reference
class LiteralBucket:
    """src/bucket.cpp:5-45 line by line (age_threshold is the literal of :16)."""

    def __init__(self, size, age_threshold=10):
        self.max_size = size
        self.age_threshold = age_threshold
        self.points, self.ages = [], []

    def size(self):
        return len(self.points)

    def add_feature(self, point, age):
        if age < self.age_threshold:
            if self.size() < self.max_size:
                self.points.append(point)
                self.ages.append(age)
            else:
                age_min = self.ages[0]
                age_min_idx = 0
                for i in range(self.size()):
                    if age < age_min:
                        age_min = age
                        age_min_idx = i
                self.points[age_min_idx] = point
                self.ages[age_min_idx] = age


def literal_bucketing(rows, cols, points, ages, bucket_size, features_per_bucket, age_threshold=10):
    """src/feature.cpp:206-253: (nh + 1) (nw + 1) buckets, indexed h * nw + w when filled and when read back."""
    nh, nw = rows // bucket_size, cols // bucket_size
    buckets = []
    for _ in range(nh + 1):
        for _ in range(nw + 1):
            buckets.append(LiteralBucket(features_per_bucket, age_threshold))
    for i in range(len(points)):
        hi = int(np.float32(points[i][1]) / np.float32(bucket_size))
        wi = int(np.float32(points[i][0]) / np.float32(bucket_size))
        buckets[hi * nw + wi].add_feature((float(points[i][0]), float(points[i][1])), int(ages[i]))
    out_p, out_a = [], []
    for hi in range(nh + 1):
        for wi in range(nw + 1):
            b = buckets[hi * nw + wi]
            out_p += b.points
            out_a += b.ages
    return np.array(out_p, np.float32).reshape(-1, 2), np.array(out_a, np.int32)


def closed_form_bucketing(rows, cols, points, ages, bucket_size, k, age_threshold=10):
    """What k_seq_bucket computes per cell: its admitted count c, its k first admitted indices and its last one."""
    nh, nw = rows // bucket_size, cols // bucket_size
    admitted = {}
    for i in range(len(points)):
        if ages[i] < age_threshold:
            idx = int(points[i][1] / np.float32(bucket_size)) * nw + int(points[i][0] / np.float32(bucket_size))
            admitted.setdefault(idx, []).append(i)
    order = []
    for hi in range(nh + 1):
        for wi in range(nw + 1):
            a = admitted.get(hi * nw + wi, [])
            order += a if len(a) <= k else [a[-1]] + a[1:k]
    order = np.array(order, np.int64)
    return np.asarray(points, np.float32).reshape(-1, 2)[order], np.asarray(ages, np.int32)[order]


def bucketing_features(rows, cols, features, bucket_size, features_per_bucket, age_threshold=10):
    """bucketingFeatures on a ref_path.FeatureSet, in place (literal_bucketing)."""
    features.points, features.ages = literal_bucketing(rows, cols, features.points, features.ages, bucket_size,
                                                       features_per_bucket, age_threshold)


def matching_features(l0, r0, l1, r1, features, backend="cv2", refill_threshold=2000, bucket_rows_divisor=10,
                      features_per_bucket=1, bucket_age_threshold=10):
    """src/visualOdometry.cpp:81-129 with the literals 2000 (:95), rows / 10 and 1 (:106-107) and bucket.cpp:16's 10 as
    keywords; the OpenCV calls and the other glue are ref_path's.  Returns (pL0, pR0, pL1, pR1, info) as
    ref_path.matching_features does."""
    from oracle import ref_path
    if features.size() < refill_threshold:
        ref_path.append_new_features(l0, features, backend)
    bucketing_features(l0.shape[0], l0.shape[1], features, l0.shape[0] // bucket_rows_divisor, features_per_bucket,
                       bucket_age_threshold)
    pts_l0 = features.points.copy()
    cm = ref_path.circular_matching(l0, r0, l1, r1, pts_l0, features, backend)
    status = ref_path.check_valid_match(cm["l0"], cm["l0_ret"], 0)
    pL0, pL1, pR0, pR1 = (ref_path.remove_invalid_points(cm[name], status) for name in ("l0", "l1", "r0", "r1"))
    features.points = pL1.copy()        # ages are NOT filtered here (SURVEY.md Appendix A item 8)
    info = dict(bucketed=pts_l0, kept_idx=cm["kept_idx"], valid=status, valid_idx=cm["kept_idx"][status])
    return pL0, pR0, pL1, pR1, info


def read_back_bound(rows, cols, divisor, k):
    bs = rows // divisor
    return (rows // bs + 1) * (cols // bs + 1) * k


def _random_admissions(rng, rows, cols, bucket_size, n):
    """Points that crowd a few cells (full buckets), sit in the last column (aliased with the next row's first) and in
    the bottom partial row, with ages around the gate."""
    nw = cols // bucket_size
    pts = rng.uniform([0, 0], [cols - 1e-3, rows - 1e-3], (n, 2)).astype(np.float32)
    hot = rng.integers(0, n, n // 2)
    pts[hot] = (rng.uniform(0, 2.5 * bucket_size, (len(hot), 2)) + [3 * bucket_size, bucket_size]).astype(np.float32)
    col = rng.integers(0, n, n // 8)
    pts[col, 0] = np.float32(nw * bucket_size) + rng.uniform(0, max(cols - nw * bucket_size, 1), len(col)).astype(np.float32)
    pts = np.minimum(pts, np.array([cols, rows], np.float32) - np.float32(1e-3))      # inside the image
    ages = rng.integers(0, 14, n).astype(np.int32)
    return pts, ages


@pytest.mark.parametrize("k", range(1, 9))
def test_bucket_and_bucketing_match_the_literal_transcription(k):
    rng = np.random.default_rng(100 + k)
    for trial in range(40):
        rows, cols = int(rng.integers(40, 400)), int(rng.integers(40, 1300))
        divisor = int(rng.integers(2, 12))
        bs = rows // divisor
        gate = int(rng.choice([0, 1, 5, 10, 1000]))
        pts, ages = _random_admissions(rng, rows, cols, bs, int(rng.integers(0, 600)))
        want_p, want_a = literal_bucketing(rows, cols, pts, ages, bs, k, gate)
        where = f"k={k} trial {trial} ({cols} x {rows} / {divisor}, gate {gate})"
        if gate == 10:                  # ref_path's bucketing has the reference's gate
            from oracle import ref_path
            fs = ref_path.FeatureSet()
            fs.points, fs.ages = pts.copy(), ages.copy()
            ref_path.bucketing_features(rows, cols, fs, bs, k)
            assert np.array_equal(fs.points, want_p) and np.array_equal(fs.ages, want_a), where
        got_p, got_a = closed_form_bucketing(rows, cols, pts, ages, bs, k, gate)
        assert np.array_equal(got_p, want_p) and np.array_equal(got_a, want_a), where
        assert len(want_p) <= read_back_bound(rows, cols, divisor, k), where


def test_a_full_bucket_overwrites_slot_zero():
    from oracle import ref_path
    for B in (LiteralBucket, ref_path.Bucket):
        b = B(3)
        for i, age in enumerate((0, 5, 2, 9, 1)):
            b.add_feature((float(i), 0.0), age)
        assert b.points == [(4.0, 0.0), (1.0, 0.0), (2.0, 0.0)] and b.ages == [1, 5, 2]
    g = LiteralBucket(2, 1)                 # age_threshold 1: only age 0 enters
    for i, age in enumerate((1, 0, 3, 0, 0)):
        g.add_feature((float(i), 0.0), age)
    assert g.points == [(4.0, 0.0), (3.0, 0.0)] and g.ages == [0, 0]


# the synthetic KITTI frame: features bucketed from its FAST corners, and the read-back bound, per (divisor, k)
FRAME_COUNTS = [(10, 1, 374, 374), (10, 2, 748, 748), (10, 4, 1490, 1496), (10, 8, 2902, 2992), (20, 1, 1449, 1449),
                (20, 4, 5795, 5796), (20, 16, 15275, 23184)]


def test_bucketed_counts_on_the_kitti_frame():
    """At 16 features per bucket the duplicated read-back of the aliased cells feeds more points than FAST found."""
    from oracle import ref_path
    img = synth.stereo_unit(seed=0)["l0"]
    corners = ref_path.fast_cv2(img)
    assert len(corners) == 15014
    for divisor, k, n, bound in FRAME_COUNTS:
        fs = ref_path.FeatureSet()
        fs.points, fs.ages = corners.copy(), np.zeros(len(corners), np.int32)
        ref_path.bucketing_features(376, 1241, fs, 376 // divisor, k)
        assert (fs.size(), read_back_bound(376, 1241, divisor, k)) == (n, bound), (divisor, k)


# ----------------------------------------------------------------------------- matchingFeatures at every keyword
def _drive(n, seed=31, w=1241, h=376):
    base = synth.stereo_unit(w, h, seed)
    fr = [(base["l0"], base["r0"])]
    for k in range(1, n):
        u = synth.stereo_unit(w, h, seed, rvec=synth.SEQ_STEP_R * k, tvec=synth.SEQ_STEP_T * k)
        fr.append((u["l1"], u["r1"]))
    return fr


CASES = [dict(features_per_bucket=3), dict(bucket_rows_divisor=20, features_per_bucket=2), dict(bucket_rows_divisor=5),
         dict(bucket_age_threshold=1), dict(bucket_age_threshold=0), dict(refill_threshold=0),
         dict(features_per_bucket=4, refill_threshold=1000)]


@pytest.mark.parametrize("prm", CASES, ids=lambda p: ",".join(f"{k}={v}" for k, v in p.items()))
def test_matching_features_keywords(prm):
    """Per frame: the refill runs exactly while fewer than refill_threshold points are live and otherwise leaves the
    FeatureSet as it is, the bucketed list is the closed form's on what the refill left, and the carried points are the
    valid L1 list with the circular check's ages."""
    pytest.importorskip("cv2")
    from oracle import ref_path
    p = dict(NEW_FIELDS, **prm)
    frames = _drive(4)
    fs = ref_path.FeatureSet()
    skipped = 0
    for k in range(1, len(frames)):
        (l0, r0), (l1, r1) = frames[k - 1], frames[k]
        points, ages = fs.points.copy(), fs.ages.copy()
        if len(points) < p["refill_threshold"]:
            new = ref_path.fast_cv2(l0, 20, True)
            points = np.concatenate([points.reshape(-1, 2), new]).astype(np.float32)
            ages = np.concatenate([ages, np.zeros(len(new), np.int32)]).astype(np.int32)
        else:
            skipped += 1
        want, want_ages = closed_form_bucketing(376, 1241, points, ages, 376 // p["bucket_rows_divisor"],
                                                p["features_per_bucket"], p["bucket_age_threshold"])
        pL0, pR0, pL1, pR1, info = matching_features(l0, r0, l1, r1, fs, "cv2", **p)
        assert np.array_equal(info["bucketed"], want), f"{prm} frame {k}: bucketed"
        # the circular check ages and compacts the bucketed ages; the validity filter leaves them alone
        assert np.array_equal(fs.points, pL1) and np.array_equal(fs.ages, (want_ages + 1)[info["kept_idx"]]), \
            f"{prm} frame {k}: FeatureSet"
        assert len(want) <= read_back_bound(376, 1241, p["bucket_rows_divisor"], p["features_per_bucket"])
    if p["refill_threshold"] <= 0 or p["bucket_age_threshold"] <= 0:
        assert len(fs.points) == 0                 # nothing ever enters (no refill, or no age passes the gate)
    if prm.get("refill_threshold") == 1000:
        assert skipped >= 1, "the live set never reached the refill threshold"


def test_default_keywords_are_ref_path():
    """At the reference's literals this file's matching_features is ref_path.matching_features bit for bit."""
    pytest.importorskip("cv2")
    from oracle import ref_path
    frames = _drive(4)
    a, b = ref_path.FeatureSet(), ref_path.FeatureSet()
    for k in range(1, len(frames)):
        x = ref_path.matching_features(*frames[k - 1], *frames[k], a, "cv2")
        y = matching_features(*frames[k - 1], *frames[k], b, "cv2", **NEW_FIELDS)
        assert all(np.array_equal(u, v) for u, v in zip(x[:4], y[:4]))
        for key in ("bucketed", "kept_idx", "valid", "valid_idx"):
            assert np.array_equal(x[4][key], y[4][key]), key
        assert np.array_equal(a.points, b.points) and np.array_equal(a.ages, b.ages)
        assert len(x[4]["bucketed"]) == 374


# ----------------------------------------------------------------------------- vo_params
def test_vo_params_layout_matches_the_header(tmp_path):
    if not shutil.which("g++"):
        pytest.skip("no host C++ compiler")
    names = [f for f, _ in capi.VoParams._fields_]
    assert names[-5:] == ["max_units", "refill_threshold", "bucket_rows_divisor", "features_per_bucket", "bucket_age_threshold"]
    src = tmp_path / "params.cpp"
    src.write_text("#include <cstdio>\n#include <cstddef>\n#include \"vo_b200.h\"\nint main() {\n"
                   "    std::printf(\"sizeof %zu\\n\", sizeof(vo_params));\n"
                   + "".join(f"    std::printf(\"{f} %zu\\n\", offsetof(vo_params, {f}));\n" for f in names) + "}\n")
    exe = tmp_path / "params"
    subprocess.run(["g++", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(ln.split(" ", 1) for ln in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(capi.VoParams)
    for f in names:
        assert int(got[f]) == getattr(capi.VoParams, f).offset, f


def test_default_params_carry_the_bucketing_literals(built):
    p = capi.VoParams()
    capi.load_library().vo_default_params(C.byref(p))
    assert {f: getattr(p, f) for f in NEW_FIELDS} == NEW_FIELDS


@pytest.mark.parametrize("field,value", [("features_per_bucket", 0), ("features_per_bucket", -3), ("bucket_rows_divisor", 0),
                                         ("bucket_rows_divisor", -10)])
def test_vo_create_refuses_empty_buckets_and_zero_divisors(built, field, value):
    """Checked before any device is touched, so the refusal is the same with or without a GPU."""
    with pytest.raises(capi.VoError) as e:
        capi.Context(0, **{field: value})
    assert e.value.code == capi.VO_E_INVALID and field in str(e.value)
