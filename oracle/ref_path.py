"""
oracle/ref_path.py -- TEST INFRASTRUCTURE ONLY (never imported by the product path).

Verbatim CPU restatement of the reference's own glue around its OpenCV calls -- quirks included
(SURVEY.md Appendix A) -- so that parity tests read like the reference's call sequence:

  FeatureSet                     reference src/feature.h:33-43
  Bucket / bucketingFeatures     reference src/bucket.cpp:5-51, src/feature.cpp:206-253
  appendNewFeatures              reference src/feature.cpp:255-262
  featureDetectionFast           reference src/feature.cpp:39-47
  deleteUnmatchFeaturesCircle    reference src/feature.cpp:76-116
  circularMatching               reference src/feature.cpp:118-148
  checkValidMatch                reference src/visualOdometry.cpp:44-61
  removeInvalidPoints            reference src/visualOdometry.cpp:63-77
  matchingFeatures               reference src/visualOdometry.cpp:81-129
  triangulate (call site)        reference src/main.cpp:170-171
  trackingFrame2Frame            reference src/visualOdometry.cpp:132-193 (mono_rotation=false branch)

The OpenCV calls themselves go either to cv2 4.13.0 (backend="cv2": the real third-party
implementation the reference links against -- this is also what bench.py times as the CPU
reference) or to the restatements in oracle/ (backend="c": lk_ref.c / fast_ref.c / pnp_ref.py).
The reference C++ itself cannot be compiled here (no OpenCV headers), see DESIGN.md.
"""
import numpy as np

try:
    import cv2
except Exception:  # pragma: no cover
    cv2 = None


class FeatureSet:
    def __init__(self):
        self.points = np.zeros((0, 2), np.float32)
        self.ages = np.zeros((0,), np.int32)

    def size(self):
        return len(self.points)

    def clear(self):
        self.points = np.zeros((0, 2), np.float32)
        self.ages = np.zeros((0,), np.int32)


# ------------------------------------------------------------------------------------ OpenCV calls
# `float confidence = 0.999;` (visualOdometry.cpp:170) reaches cv::solvePnPRansac as (double)0.999f
PNP_CONFIDENCE = float(np.float32(0.999))
# the literals of the reference's calcOpticalFlowPyrLK call (feature.cpp:127-139: 21 x 21 window, maxLevel 3, 30
# iterations, epsilon 0.01, minEigThreshold 0.001) are the defaults of the LK keywords below (max_level, max_iters,
# epsilon, min_eig); the window stays 21 x 21


def fast_cv2(img, threshold=20, nonmax=True):
    fd = cv2.FastFeatureDetector_create(threshold, nonmax)
    kps = fd.detect(img)
    return np.array([k.pt for k in kps], np.float32).reshape(-1, 2)


def lk_cv2(prev, nxt, pts, max_level=3, max_iters=30, epsilon=0.01, min_eig=0.001, with_err=False):
    if len(pts) == 0:
        return (np.zeros((0, 2), np.float32), np.zeros((0,), np.uint8)) + ((np.zeros((0,), np.float32),) if with_err else ())
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, max_iters, epsilon)
    o, s, e = cv2.calcOpticalFlowPyrLK(prev, nxt, np.ascontiguousarray(pts, np.float32).reshape(-1, 1, 2), None,
                                       criteria=crit, winSize=(21, 21), maxLevel=max_level, flags=0, minEigThreshold=min_eig)
    return (o.reshape(-1, 2), s.ravel()) + ((e.ravel(),) if with_err else ())


def lk_c(prev, nxt, pts, max_level=3, max_iters=30, epsilon=0.01, min_eig=0.001, with_err=False):
    from . import cref
    o, s, e = cref.lk_track(prev, nxt, pts, max_level=max_level, max_count=max_iters, epsilon=epsilon, min_eig=min_eig)
    return (o, s) + ((e,) if with_err else ())


def fast_c(img, threshold=20, nonmax=True):
    from . import cref
    return cref.fast_detect(img, threshold, nonmax)[0]


def _backend(name):
    if name == "cv2":
        return fast_cv2, lk_cv2
    return fast_c, lk_c


# ------------------------------------------------------------------------------------ glue
def delete_unmatch_features_circle(p0, p1, p2, p3, p0r, s0, s1, s2, s3, ages):
    """feature.cpp:76-116.  ages is incremented for ALL entries first, then everything is
    compacted in lock-step; points0_return is not part of the negative-coordinate test.
    Returns the compacted arrays, the modified status3 and the surviving original indices."""
    ages = np.asarray(ages, np.int32) + 1
    n = len(s3)
    neg = (p0[:, 0] < 0) | (p0[:, 1] < 0) | (p1[:, 0] < 0) | (p1[:, 1] < 0) | \
          (p2[:, 0] < 0) | (p2[:, 1] < 0) | (p3[:, 0] < 0) | (p3[:, 1] < 0)
    bad = (s3 == 0) | (s2 == 0) | (s1 == 0) | (s0 == 0) | neg
    s3 = s3.copy()
    s3[neg] = 0
    keep = np.nonzero(~bad)[0]
    # ages may be longer/shorter than the point vectors (Appendix A item 8): erase() works by
    # position, so only the first n entries participate and any excess tail is carried over
    if len(ages) >= n:
        ages_out = np.concatenate([ages[:n][keep], ages[n:]])
    else:
        ages_out = ages[keep[keep < len(ages)]]
    return p0[keep], p1[keep], p2[keep], p3[keep], p0r[keep], s3, ages_out, keep.astype(np.int32)


def circular_matching(l0, r0, l1, r1, pts_l0, features, backend="cv2", max_level=3, max_iters=30, epsilon=0.01,
                      min_eig=0.001):
    """feature.cpp:118-148: ring L0->R0->R1->L1->L0 then deleteUnmatchFeaturesCircle.
    Returns dict with the five compacted vectors, raw per-call outputs/status, kept indices."""
    _, lk_fn = _backend(backend)
    lk = lambda a, b, p: lk_fn(a, b, p, max_level=max_level, max_iters=max_iters, epsilon=epsilon, min_eig=min_eig)
    pts_l0 = np.ascontiguousarray(pts_l0, np.float32).reshape(-1, 2)
    pr0, s0 = lk(l0, r0, pts_l0)
    pr1, s1 = lk(r0, r1, pr0)
    pl1, s2 = lk(r1, l1, pr1)
    pl0r, s3 = lk(l1, l0, pl1)
    raw = dict(r0=pr0, r1=pr1, l1=pl1, l0_ret=pl0r, status=np.stack([s0, s1, s2, s3]) if len(pts_l0) else np.zeros((4, 0), np.uint8))
    a, b, c, d, e, s3m, ages, keep = delete_unmatch_features_circle(pts_l0, pr0, pr1, pl1, pl0r, s0, s1, s2, s3, features.ages)
    features.ages = ages
    return dict(l0=a, r0=b, r1=c, l1=d, l0_ret=e, kept_idx=keep, raw=raw)


def check_valid_match(points, points_return, threshold=0):
    """visualOdometry.cpp:44-61: `int offset` truncates the float max-abs difference."""
    d = np.maximum(np.abs(points[:, 0] - points_return[:, 0]), np.abs(points[:, 1] - points_return[:, 1]))
    offset = d.astype(np.float32).astype(np.int32)          # float -> int truncation toward zero
    return ~(offset > threshold)


def remove_invalid_points(points, status):
    return points[np.asarray(status, bool)]


class Bucket:
    """bucket.cpp:5-51 (the 'replace youngest' loop compares the incoming age with itself, so a
    full bucket always overwrites slot 0)."""

    def __init__(self, size):
        self.max_size = size
        self.points = []
        self.ages = []

    def add_feature(self, point, age):
        if age < 10:
            if len(self.points) < self.max_size:
                self.points.append(point); self.ages.append(age)
            else:
                age_min = self.ages[0]
                age_min_idx = 0
                for i in range(len(self.points)):
                    if age < age_min:
                        age_min = age
                        age_min_idx = i
                self.points[age_min_idx] = point
                self.ages[age_min_idx] = age


def bucketing_features(rows, cols, features, bucket_size, features_per_bucket):
    """feature.cpp:206-253: (nh+1)*(nw+1) buckets but index stride nw -> aliasing + duplicated
    read-back (SURVEY.md row A4).  Coordinates outside the image would index past the vector in
    the reference (UB); here they raise."""
    nh = rows // bucket_size
    nw = cols // bucket_size
    buckets = [Bucket(features_per_bucket) for _ in range((nh + 1) * (nw + 1))]
    pts = features.points
    ages = features.ages
    for i in range(len(pts)):
        bh = int(np.float32(pts[i][1]) / np.float32(bucket_size))     # float / int -> float -> int
        bw = int(np.float32(pts[i][0]) / np.float32(bucket_size))
        idx = bh * nw + bw
        buckets[idx].add_feature((float(pts[i][0]), float(pts[i][1])), int(ages[i]))
    out_p, out_a = [], []
    for ih in range(nh + 1):
        for iw in range(nw + 1):
            b = buckets[ih * nw + iw]
            out_p.extend(b.points); out_a.extend(b.ages)
    features.points = np.array(out_p, np.float32).reshape(-1, 2)
    features.ages = np.array(out_a, np.int32)


def append_new_features(img, features, backend="cv2"):
    fast, _ = _backend(backend)
    new = fast(img, 20, True)
    features.points = np.concatenate([features.points.reshape(-1, 2), new]).astype(np.float32)
    features.ages = np.concatenate([features.ages, np.zeros(len(new), np.int32)]).astype(np.int32)


def matching_features(l0, r0, l1, r1, features, backend="cv2", max_level=3, max_iters=30, epsilon=0.01, min_eig=0.001,
                      circ_threshold=0):
    """visualOdometry.cpp:81-129.  Returns (pL0, pR0, pL1, pR1, info).  The keywords replace the reference's literals
    (the LK call's, and checkValidMatch's threshold 0 at :120)."""
    if features.size() < 2000:
        append_new_features(l0, features, backend)
    bucket_size = l0.shape[0] // 10
    bucketing_features(l0.shape[0], l0.shape[1], features, bucket_size, 1)
    pts_l0 = features.points.copy()
    cm = circular_matching(l0, r0, l1, r1, pts_l0, features, backend, max_level=max_level, max_iters=max_iters,
                           epsilon=epsilon, min_eig=min_eig)
    status = check_valid_match(cm["l0"], cm["l0_ret"], circ_threshold)
    pL0 = remove_invalid_points(cm["l0"], status)
    pL1 = remove_invalid_points(cm["l1"], status)
    pR0 = remove_invalid_points(cm["r0"], status)
    pR1 = remove_invalid_points(cm["r1"], status)
    features.points = pL1.copy()        # ages are NOT filtered here (Appendix A item 8)
    info = dict(bucketed=pts_l0, kept_idx=cm["kept_idx"], valid=status, valid_idx=cm["kept_idx"][status])
    return pL0, pR0, pL1, pR1, info


def triangulate(P_l, P_r, pts_l, pts_r, backend="cv2"):
    """main.cpp:170-171: triangulatePoints + convertPointsFromHomogeneous -> (N,3) float32."""
    if backend == "cv2":
        if len(pts_l) == 0:
            return np.zeros((0, 3), np.float32)
        X4 = cv2.triangulatePoints(P_l, P_r, np.ascontiguousarray(pts_l, np.float32).T.copy(),
                                   np.ascontiguousarray(pts_r, np.float32).T.copy())
        return cv2.convertPointsFromHomogeneous(X4.T.copy()).reshape(-1, 3)
    from . import pnp_ref
    return pnp_ref.triangulate(P_l, P_r, pts_l, pts_r)


def tracking_frame2frame(P_l, pts_l0, pts_l1, X, translation, backend="cv2", iterations=500, reproj=0.5,
                         confidence=PNP_CONFIDENCE):
    """visualOdometry.cpp:132-193 with mono_rotation=false (what main.cpp:181 passes); the keywords replace the literals
    of its solvePnPRansac call (:168-170).  Returns (rotation 3x3 f64, translation 3 f64, inlier indices int32, rvec)."""
    K = np.ascontiguousarray(P_l[:, :3], np.float32)
    if backend == "cv2":
        dist = np.zeros((4, 1), np.float64)
        rvec = np.zeros((3, 1), np.float64)
        tvec = np.asarray(translation, np.float64).reshape(3, 1).copy()
        ok, rvec, tvec, inl = cv2.solvePnPRansac(
            np.ascontiguousarray(X, np.float32).reshape(-1, 1, 3), np.ascontiguousarray(pts_l1, np.float32).reshape(-1, 1, 2),
            K, dist, rvec, tvec, True, iterations, reproj, confidence, None, cv2.SOLVEPNP_ITERATIVE)
        R, _ = cv2.Rodrigues(rvec)
        inl = np.zeros((0,), np.int32) if inl is None else inl.ravel().astype(np.int32)
        return R, tvec.ravel(), inl, rvec.ravel()
    from . import pnp_ref
    res = pnp_ref.solve_pnp_ransac(X, pts_l1, K, np.zeros(3), translation, iterations=iterations, reproj=reproj,
                                   confidence=confidence)
    return pnp_ref.rodrigues(res["rvec"]), res["tvec"], res["inliers"], res["rvec"]


def rotation_matrix_to_euler_angles(R):
    """utils.cpp:107-131 (sy is a float there)."""
    sy = np.float32(np.sqrt(R[0, 0] * R[0, 0] + R[1, 0] * R[1, 0]))
    if not sy < 1e-6:
        return np.array([np.arctan2(R[2, 1], R[2, 2]), np.arctan2(-R[2, 0], float(sy)), np.arctan2(R[1, 0], R[0, 0])], np.float32)
    return np.array([np.arctan2(-R[1, 2], R[1, 1]), np.arctan2(-R[2, 0], float(sy)), 0.0], np.float32)


def integrate_pose(frame_pose, R, t):
    """main.cpp:196-208 + utils.cpp:57-91: Euler gate (all |angles| < 0.1), then frame_pose *= [R|t]^-1
    when 0.05 < |t| < 10."""
    e = rotation_matrix_to_euler_angles(R)
    if not (abs(e[1]) < 0.1 and abs(e[0]) < 0.1 and abs(e[2]) < 0.1):
        return frame_pose
    T = np.eye(4); T[:3, :3] = R; T[:3, 3] = t
    scale = np.sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2])
    if 0.05 < scale < 10:
        return frame_pose @ np.linalg.inv(T)
    return frame_pose
