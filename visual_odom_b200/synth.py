"""KITTI-shaped synthetic stereo work units (SURVEY.md section 8d "Synthetic inputs").

There is no network and no dataset in this environment, so every test / benchmark input is
generated here, deterministically from a seed.  cv2 is used only as an image library
(resize / blur / remap); nothing in here is on the measured path.

scene "v1": three fronto-parallel textured planes (stereo disparities 4 / 12 / 40 px at KITTI-00
intrinsics) seen by a calibrated stereo rig that moves by a known ego-motion between t0 and t1;
each of the four views (L0, R0, L1, R1) is rendered through the exact plane homography and gets
independent N(0,1) sensor noise.  scene "v0": pure-translation crops of one texture.
"""
import numpy as np
import cv2

KITTI00 = dict(fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, bf=-386.1448)      # calibration/kitti00.yaml:8-14
ZED = dict(fx=684.367919921875 * 1.5, fy=684.367919921875 * 1.5, cx=960.0, cy=540.0,
           bf=-82.12415128946304 * 1.5)                                               # calibration/zed.yaml scaled to 1920x1080
# Stereo rigs in the terms of an ORB-SLAM2 settings file (LEFT / RIGHT .K, .D, .R, .P; P is 3 x 4), for rectification
# (vo_seq_rectify, vo_mseq_rectify): EuRoC's cam0 / cam1 as ORB-SLAM2's EuRoC.yaml gives them, and a KITTI-raw-like colour
# pair (5 coefficients, small rectifying rotations).
_EUROC_CAM0 = dict(
    K=[458.654, 0.0, 367.215, 0.0, 457.296, 248.375, 0.0, 0.0, 1.0],
    D=[-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0],
    R=[0.999966347530033, -0.001422739138722922, 0.008079580483432283, 0.001365741834644127, 0.9999741760894847,
       0.007055629199258132, -0.008089410156878961, -0.007044357138835809, 0.9999424675829176],
    P=[435.2046959714599, 0, 367.4517211914062, 0, 0, 435.2046959714599, 252.2008514404297, 0, 0, 0, 1, 0])
_EUROC_CAM1 = dict(
    K=[457.587, 0.0, 379.999, 0.0, 456.134, 255.238, 0.0, 0.0, 1],
    D=[-0.28368365, 0.07451284, -0.00010473, -3.55590700e-05, 0.0],
    R=[0.9999633526194376, -0.003625811871560086, 0.007755443660172947, 0.003680398547259526, 0.9999684752771629,
       -0.007035845251224894, -0.007729688520722713, 0.007064130529506649, 0.999945173484644],
    P=[435.2046959714599, 0, 367.4517211914062, -47.90639384423901, 0, 435.2046959714599, 252.2008514404297, 0, 0, 0, 1, 0])
_KITTI_RAW_LEFT = dict(
    K=[959.791, 0.0, 696.0217, 0.0, 956.9251, 224.1806, 0.0, 0.0, 1.0],
    D=[-0.3691481, 0.1968681, 0.001353473, 0.0005677587, -0.06770705],
    R=[0.9999239, 0.00983776, -0.007445048, -0.009869795, 0.9999421, -0.004278459, 0.007402527, 0.004351614, 0.9999631],
    P=[721.5377, 0.0, 609.5593, 44.85728, 0.0, 721.5377, 172.854, 0.2163791, 0.0, 0.0, 1.0, 0.002745884])
_KITTI_RAW_RIGHT = dict(
    _KITTI_RAW_LEFT,
    R=[0.9999805, -0.006070, 0.001402, 0.006073, 0.9999793, -0.002209, -0.001389, 0.002218, 0.9999966],
    P=[721.5377, 0.0, 609.5593, -339.5242, 0.0, 721.5377, 172.854, 2.199936, 0.0, 0.0, 1.0, 0.002729905])
RECTIFY_CAMS = {"euroc_cam0": _EUROC_CAM0, "euroc_cam1": _EUROC_CAM1, "kitti_raw_left": _KITTI_RAW_LEFT,
                "kitti_raw_right": _KITTI_RAW_RIGHT}


def rectify_cam_matrices(c):
    """(K 3x3, D, R 3x3, P 3x4) float64 of one RECTIFY_CAMS entry."""
    return (np.asarray(c["K"], np.float64).reshape(3, 3), np.asarray(c["D"], np.float64),
            np.asarray(c["R"], np.float64).reshape(3, 3), np.asarray(c["P"], np.float64).reshape(3, -1))


def rectify_rig(left, right):
    """{"left": (K, D, R, P), "right": (...)} of two RECTIFY_CAMS names: what Context.seq_rectify / mseq_rectify take."""
    return {"left": rectify_cam_matrices(RECTIFY_CAMS[left]), "right": rectify_cam_matrices(RECTIFY_CAMS[right])}


EGO_RVEC = np.array([0.004, -0.02, 0.001])
EGO_T = np.array([0.03, -0.01, -0.9])


def proj_matrices(cal=KITTI00):
    """P_l, P_r exactly as reference src/main.cpp:73-74 builds them (3x4 float32)."""
    fx, fy, cx, cy, bf = (np.float32(cal[k]) for k in ("fx", "fy", "cx", "cy", "bf"))
    P_l = np.array([[fx, 0, cx, 0], [0, fy, cy, 0], [0, 0, 1, 0]], np.float32)
    P_r = np.array([[fx, 0, cx, bf], [0, fy, cy, 0], [0, 0, 1, 0]], np.float32)
    return P_l, P_r


def texture(h, w, seed, margin=96):
    rng = np.random.default_rng(seed)
    lo = rng.integers(0, 256, size=((h + 2 * margin) // 4 + 2, (w + 2 * margin) // 4 + 2)).astype(np.uint8)
    up = cv2.resize(lo, (w + 2 * margin, h + 2 * margin), interpolation=cv2.INTER_CUBIC)
    return cv2.GaussianBlur(up, (0, 0), 1.0)


def _rodrigues(r):
    R, _ = cv2.Rodrigues(np.asarray(r, np.float64).reshape(3, 1))
    return R


def stereo_unit(w=1241, h=376, seed=0, cal=KITTI00, scene="v1", noise=1.0, rvec=EGO_RVEC, tvec=EGO_T, sky=0.0):
    """Returns dict(l0, r0, l1, r1 : uint8 HxW, P_l, P_r, K, rvec, tvec).

    sky > 0 (scene "v1" only) overwrites the top `sky` fraction of L0's rows with a textured band at infinity: in each
    view it is drawn through the rotation-only homography K R K^-1, so the left and right images of one time carry the
    same pixels there, sensor noise included (zero disparity), and t1 sees the band rotated by `rvec` only.  The default
    0 leaves every image, and the noise drawn for it, as before."""
    P_l, P_r = proj_matrices(cal)
    K = P_l[:, :3].astype(np.float64)
    rng = np.random.default_rng(1000 + seed)
    margin = 96
    if sky and scene != "v1":
        raise ValueError("sky needs scene 'v1'")
    sky_masks = []
    if scene == "v0":
        T = texture(h, w, seed, margin)
        def crop(dx, dy):
            return T[margin + dy:margin + dy + h, margin + dx:margin + dx + w].copy()
        views = [crop(0, 0), crop(6, 0), crop(-2, -1), crop(4, -1)]          # L0, R0, L1, R1
    else:
        disp = [4.0, 12.0, 40.0]
        Z = [-float(cal["bf"]) / d for d in disp]
        # L0 band membership: far plane on top, near plane at the bottom
        bands = [(0, int(h * 0.40)), (int(h * 0.40), int(h * 0.72)), (int(h * 0.72), h)]
        texs = [texture(h, w, seed * 3 + k, margin) for k in range(3)]
        base = float(cal["bf"]) / float(cal["fx"])            # X_r = X_l + (base, 0, 0)
        R1 = _rodrigues(rvec)
        poses = [(np.eye(3), np.zeros(3)),                    # L0
                 (np.eye(3), np.array([base, 0, 0])),         # R0
                 (R1, np.asarray(tvec, np.float64)),          # L1:  X_1 = R X_0 + t
                 (R1, np.asarray(tvec, np.float64) + np.array([base, 0, 0]))]   # R1
        uu, vv = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
        pix = np.stack([uu.ravel(), vv.ravel(), np.ones(w * h)], 0)
        Kinv = np.linalg.inv(K)
        sky_tex = texture(h, w, 10007 + seed, margin) if sky > 0 else None
        views = []
        for (R, t) in poses:
            img = np.zeros((h, w), np.uint8)
            filled = np.zeros((h, w), bool)
            for k in (2, 1, 0):                                # nearest plane wins
                n = np.array([0.0, 0.0, 1.0])
                H = K @ (R + np.outer(t, n) / Z[k]) @ Kinv   # L0 pixel -> view pixel
                p0 = np.linalg.inv(H) @ pix
                x0 = (p0[0] / p0[2]).reshape(h, w)
                y0 = (p0[1] / p0[2]).reshape(h, w)
                inside = (y0 >= bands[k][0]) & (y0 < bands[k][1]) & ~filled
                m = cv2.remap(texs[k], (x0 + margin).astype(np.float32), (y0 + margin).astype(np.float32),
                              cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)
                img[inside] = m[inside]
                filled |= inside
            if not filled.all():                               # slivers between bands: far plane
                H = K @ (R + np.outer(t, np.array([0.0, 0.0, 1.0])) / Z[0]) @ Kinv
                p0 = np.linalg.inv(H) @ pix
                m = cv2.remap(texs[0], ((p0[0] / p0[2]).reshape(h, w) + margin).astype(np.float32),
                              ((p0[1] / p0[2]).reshape(h, w) + margin).astype(np.float32),
                              cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)
                img[~filled] = m[~filled]
            if sky > 0:                                        # the band at infinity: L0 pixel -> view pixel is K R K^-1
                p0 = np.linalg.inv(K @ R @ Kinv) @ pix
                x0 = (p0[0] / p0[2]).reshape(h, w)
                y0 = (p0[1] / p0[2]).reshape(h, w)
                inside = y0 < sky * h
                m = cv2.remap(sky_tex, (x0 + margin).astype(np.float32),
                              (y0 + margin).astype(np.float32), cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)
                img[inside] = m[inside]
                sky_masks.append(inside)
            views.append(img)
    out = []
    for v in views:
        if noise > 0:
            v = np.clip(v.astype(np.int32) + np.rint(rng.normal(0, noise, v.shape)).astype(np.int32), 0, 255).astype(np.uint8)
        out.append(np.ascontiguousarray(v))
    if sky > 0:                                                # right = left in the band, noise included
        for left, right in ((0, 1), (2, 3)):
            assert np.array_equal(sky_masks[left], sky_masks[right])
            out[right][sky_masks[left]] = out[left][sky_masks[left]]
    return dict(l0=out[0], r0=out[1], l1=out[2], r1=out[3], P_l=P_l, P_r=P_r,
                K=P_l[:, :3].copy(), rvec=np.asarray(rvec, np.float64), tvec=np.asarray(tvec, np.float64))


SEQ_STEP_R = np.array([0.001, -0.004, 0.0005])          # per-frame ego-motion of the synthetic drives
SEQ_STEP_T = np.array([0.01, -0.003, -0.2])


def _rodrigues_np(r):
    r = np.asarray(r, np.float64)
    th = float(np.linalg.norm(r))
    if th == 0.0:
        return np.eye(3)
    k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1.0 - np.cos(th)) * (Kx @ Kx)


def blob_sequence(w=1241, h=376, seed=4, n_points=160, n_frames=24, sharp=lambda k: k < 3 or k >= 18,
                  cal=KITTI00, step_r=SEQ_STEP_R, step_t=SEQ_STEP_T):
    """A sparse drive on which features live for many frames: n_points isolated world points (X in U(-25, 25),
    Y in U(-4, 3), Z in U(10, 45) m), each drawn as a Gaussian blob at its exact projection on a flat background of 100
    with N(0, 1) noise, rounded to u8.  Frame k is rendered at rotation Rodrigues(k step_r) and translation k step_t.
    Sharp frames (sharp(k) true: sigma 1.3 px, amplitude +80) fire FAST; soft frames (sigma 3.5 px, amplitude +50: the
    centre-to-ring contrast stays below FAST's threshold of 20) detect nothing new while LK still tracks the blobs, so
    through a soft stretch the tracked features age by one per frame.  numpy only, deterministic in the seed.
    Returns (P_l, P_r, frames) with frames[k] = (left, right)."""
    P_l, P_r = proj_matrices(cal)
    K = P_l[:, :3].astype(np.float64)
    base = float(cal["bf"]) / float(cal["fx"])              # X_r = X_l + (base, 0, 0)
    rng = np.random.default_rng(seed)
    X = np.stack([rng.uniform(-25, 25, n_points), rng.uniform(-4, 3, n_points), rng.uniform(10, 45, n_points)], 1)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    r = 15                                                  # blob support: +-15 px (4.3 sigma of a soft blob)

    def render(R, t, is_sharp, noise_seed):
        Xc = X @ R.T + t
        u = Xc[:, 0] / Xc[:, 2] * K[0, 0] + K[0, 2]
        v = Xc[:, 1] / Xc[:, 2] * K[1, 1] + K[1, 2]
        s, A = (1.3, 80.0) if is_sharp else (3.5, 50.0)
        img = np.full((h, w), 100.0)
        for a, b in zip(u, v):
            x0, x1, y0, y1 = int(max(0, a - r)), int(min(w, a + r + 1)), int(max(0, b - r)), int(min(h, b + r + 1))
            if x0 >= x1 or y0 >= y1:
                continue
            img[y0:y1, x0:x1] += A * np.exp(-((xx[y0:y1, x0:x1] - a) ** 2 + (yy[y0:y1, x0:x1] - b) ** 2) / (2 * s * s))
        img += np.random.default_rng(noise_seed).normal(0, 1.0, img.shape)
        return np.clip(np.rint(img), 0, 255).astype(np.uint8)

    frames = []
    for k in range(n_frames):
        R = _rodrigues_np(np.asarray(step_r, np.float64) * k)
        t = np.asarray(step_t, np.float64) * k
        frames.append((render(R, t, sharp(k), (seed, k, 0)), render(R, t + np.array([base, 0.0, 0.0]), sharp(k), (seed, k, 1))))
    return P_l, P_r, frames


def select_features(corners, n):
    """Even-stride selection over the raster-ordered FAST list (SURVEY.md 8d "Features")."""
    corners = np.asarray(corners, np.float32).reshape(-1, 2)
    m = len(corners)
    if m == 0 or n <= 0:
        return corners[:0]
    if n >= m:
        return corners.copy()
    idx = (np.arange(n, dtype=np.int64) * (m - 1)) // (n - 1) if n > 1 else np.array([0])
    return corners[idx]


def pnp_stress_set(n=1500, sigma=0.15, outlier_frac=0.3, seed=0, cal=KITTI00, rvec=EGO_RVEC, tvec=EGO_T):
    """3-D points + noisy projections + gross outliers (SURVEY.md 8d "PnP stress set")."""
    rng = np.random.default_rng(seed)
    P_l, _ = proj_matrices(cal)
    K = P_l[:, :3].astype(np.float64)
    X = np.stack([rng.uniform(-30, 30, n), rng.uniform(-3, 6, n), rng.uniform(6, 80, n)], 1).astype(np.float32)
    R = _rodrigues(rvec)
    Xc = X.astype(np.float64) @ R.T + np.asarray(tvec, np.float64)
    x = np.stack([Xc[:, 0] / Xc[:, 2] * K[0, 0] + K[0, 2], Xc[:, 1] / Xc[:, 2] * K[1, 1] + K[1, 2]], 1)
    x += rng.normal(0, sigma, x.shape)
    out = rng.random(n) < outlier_frac
    x[out] += rng.uniform(-15, 15, (int(out.sum()), 2))
    return X, x.astype(np.float32), P_l[:, :3].copy(), out


def essential_stress_set(n, sigma, outlier_frac, seed, cal=KITTI00, rvec=EGO_RVEC, tvec=EGO_T):
    """Image points of n world points before / after the ego-motion (pixel noise sigma on both, a fraction of gross
    outliers in the second view) + the (focal, principal point) the reference's mono branch reads from P_l as floats
    (reference src/visualOdometry.cpp:144-145).  Returns (p_t0, p_t1, focal, pp)."""
    rng = np.random.default_rng(seed)
    P_l, _ = proj_matrices(cal)
    K = P_l[:, :3].astype(np.float64)
    X = np.stack([rng.uniform(-30, 30, n), rng.uniform(-3, 6, n), rng.uniform(6, 80, n)], 1)
    x0 = np.stack([X[:, 0] / X[:, 2] * K[0, 0] + K[0, 2], X[:, 1] / X[:, 2] * K[1, 1] + K[1, 2]], 1)
    Xc = X @ _rodrigues(rvec).T + np.asarray(tvec, np.float64)
    x1 = np.stack([Xc[:, 0] / Xc[:, 2] * K[0, 0] + K[0, 2], Xc[:, 1] / Xc[:, 2] * K[1, 1] + K[1, 2]], 1)
    x0 += rng.normal(0, sigma, x0.shape); x1 += rng.normal(0, sigma, x1.shape)
    o = rng.random(n) < outlier_frac
    x1[o] += rng.uniform(-15, 15, (int(o.sum()), 2))
    return x0.astype(np.float32), x1.astype(np.float32), float(np.float32(K[0, 0])), (float(np.float32(K[0, 2])), float(np.float32(K[1, 2])))
