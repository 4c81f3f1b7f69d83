"""Image pairs and LK starts on which every window from 3x3 to 32x32 is checked (tests/test_oracle_lk_windows.py pins the
oracle to cv2 on them, tests/test_gpu_lk_windows.py the GPU to both): a blurred-noise image and a slightly rotated and
shifted copy, a KITTI-size stereo pair with starts up to 40 px outside the image, and saturated 2x2 blocks of 0 / 255; and
the reference's glue around calcOpticalFlowPyrLK at any window, against which the GPU's modes are checked."""
import numpy as np

from visual_odom_b200 import synth

WINDOWS = tuple(range(3, 33))


def _blur(a):
    """[1 4 6 4 1] / 16 along both axes, edges replicated"""
    k = np.array([1, 4, 6, 4, 1], np.float64) / 16
    for axis in (0, 1):
        p = np.pad(a, [(2, 2) if ax == axis else (0, 0) for ax in (0, 1)], mode="edge")
        a = sum(k[i] * np.take(p, np.arange(i, i + a.shape[axis]), axis=axis) for i in range(5))
    return a


def _warp(a, angle, shift):
    """a sampled bilinearly at the points that a rotation by `angle` about the centre plus `shift` maps the output to"""
    h, w = a.shape
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    c, s = np.cos(angle), np.sin(angle)
    xc, yc = x - w / 2 - shift[0], y - h / 2 - shift[1]
    sx = np.clip(c * xc + s * yc + w / 2, 0, w - 1.001)
    sy = np.clip(-s * xc + c * yc + h / 2, 0, h - 1.001)
    x0, y0 = np.floor(sx).astype(int), np.floor(sy).astype(int)
    fx, fy = sx - x0, sy - y0
    return ((1 - fx) * (1 - fy) * a[y0, x0] + fx * (1 - fy) * a[y0, x0 + 1] + (1 - fx) * fy * a[y0 + 1, x0]
            + fx * fy * a[y0 + 1, x0 + 1])


def _starts(rng, w, h, n_in, n_out, margin):
    inside = np.stack([rng.uniform(2, w - 2, n_in), rng.uniform(2, h - 2, n_in)], 1)
    anywhere = np.stack([rng.uniform(-margin, w + margin, n_out), rng.uniform(-margin, h + margin, n_out)], 1)
    return np.concatenate([inside, anywhere]).astype(np.float32)


def noise_pair(seed=3):
    """320 x 240 blurred noise and a copy rotated by 0.6 degrees and shifted by (2.3, -1.6); 1500 starts, 200 of them
    anywhere within 40 px of the image"""
    rng = np.random.default_rng(seed)
    a = _blur(_blur(rng.uniform(0, 255, (240, 320))))
    a = (a - a.min()) / (a.max() - a.min()) * 255
    b = _warp(a, np.deg2rad(0.6), (2.3, -1.6))
    return np.round(a).astype(np.uint8), np.round(b).astype(np.uint8), _starts(rng, 320, 240, 1300, 200, 40)


def stereo_pair(seed=5):
    """synth.stereo_unit(1241, 376, seed) l0 -> r0; 700 FAST corners and 100 starts up to 40 px outside the image"""
    from oracle import cref
    u = synth.stereo_unit(1241, 376, seed)
    corners, _ = cref.fast_detect(u["l0"])
    rng = np.random.default_rng(seed)
    out = np.stack([rng.uniform(-40, 1241 + 40, 100), rng.uniform(-40, 376 + 40, 100)], 1).astype(np.float32)
    return u["l0"], u["r0"], np.concatenate([synth.select_features(corners, 700), out])


def block_pair(w=300, h=200, seed=8, n=800):
    """saturated 2 x 2 blocks of 0 / 255 and the same blocks shifted by (1, 2); n starts, an eighth of them within 40 px
    outside the image"""
    rng = np.random.default_rng(seed)
    a = np.kron(rng.integers(0, 2, (h // 2, w // 2)) * 255, np.ones((2, 2))).astype(np.uint8)
    b = np.roll(a, (2, 1), axis=(0, 1))
    return a, b, _starts(rng, w, h, n - n // 8, n // 8, 40)


SCENES = {"noise": noise_pair, "stereo": stereo_pair, "blocks": block_pair}


# ------------------------------------------------------------------------------------ the reference's glue at a window
# oracle/ref_path.py restates the reference's glue around calcOpticalFlowPyrLK with its Size(21,21) literal; these are the
# same calls at a win x win window, built from ref_path's own pieces
def lk(prev, nxt, pts, win, backend="cv2", max_level=3, max_iters=30, epsilon=0.01, min_eig=0.001):
    """one calcOpticalFlowPyrLK call (flags 0, err requested) on cv2 or on the oracle: (positions, status, err)"""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    if backend != "cv2":
        from oracle import cref
        return cref.lk_track(prev, nxt, pts, win=win, max_level=max_level, max_count=max_iters, epsilon=epsilon,
                             min_eig=min_eig)
    import cv2
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, max_iters, epsilon)
    o, s, e = cv2.calcOpticalFlowPyrLK(prev, nxt, pts.reshape(-1, 1, 2), None, criteria=crit, winSize=(win, win),
                                       maxLevel=max_level, flags=0, minEigThreshold=min_eig)
    return o.reshape(-1, 2), s.ravel(), e.ravel()


def circular_matching(l0, r0, l1, r1, pts_l0, features, win, backend="cv2"):
    """ref_path.circular_matching (feature.cpp:118-148) at a win x win window"""
    from oracle import ref_path
    pts_l0 = np.ascontiguousarray(pts_l0, np.float32).reshape(-1, 2)
    pr0, s0, _ = lk(l0, r0, pts_l0, win, backend)
    pr1, s1, _ = lk(r0, r1, pr0, win, backend)
    pl1, s2, _ = lk(r1, l1, pr1, win, backend)
    pl0r, s3, _ = lk(l1, l0, pl1, win, backend)
    raw = dict(r0=pr0, r1=pr1, l1=pl1, l0_ret=pl0r, status=np.stack([s0, s1, s2, s3]))
    a, b, c, d, e, _, ages, keep = ref_path.delete_unmatch_features_circle(pts_l0, pr0, pr1, pl1, pl0r, s0, s1, s2, s3,
                                                                           features.ages)
    features.ages = ages
    return dict(l0=a, r0=b, r1=c, l1=d, l0_ret=e, kept_idx=keep, raw=raw)


def matching_features(l0, r0, l1, r1, features, win, backend="cv2"):
    """ref_path.matching_features (visualOdometry.cpp:81-129, the reference's other literals) at a win x win window"""
    from oracle import ref_path
    if features.size() < 2000:
        ref_path.append_new_features(l0, features, backend)
    ref_path.bucketing_features(l0.shape[0], l0.shape[1], features, l0.shape[0] // 10, 1)
    pts_l0 = features.points.copy()
    cm = circular_matching(l0, r0, l1, r1, pts_l0, features, win, backend)
    status = ref_path.check_valid_match(cm["l0"], cm["l0_ret"], 0)
    pL0, pR0, pL1, pR1 = (ref_path.remove_invalid_points(cm[k], status) for k in ("l0", "r0", "l1", "r1"))
    features.points = pL1.copy()        # ages are NOT filtered here
    return pL0, pR0, pL1, pR1, dict(bucketed=pts_l0, kept_idx=cm["kept_idx"], valid=status)
