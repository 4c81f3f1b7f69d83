"""Stereo triangulation at the disparities where it goes wrong: zero, a few float ulps, around the point where the DLT's
w crosses FLT_EPSILON (cv::convertPointsFromHomogeneous divides only above it), sub-pixel, negative, with a vertical
mismatch, far outside the image, and one point alone.  Both the oracle (oracle/pnp_ref.py) and the kernels' own math
(pnp_math.cuh compiled for the host) are pinned bit for bit to cv2.triangulatePoints + convertPointsFromHomogeneous, and
the homogeneous column and the 3-D point to an independent float64 computation, so that a fault cv2 and the oracle
shared would show too."""
import ctypes as C

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from oracle import pnp_ref as P
from visual_odom_b200 import synth

EPS = np.float32(np.finfo(np.float32).eps)            # FLT_EPSILON
CALS = {"kitti": (synth.KITTI00, 1241, 376), "zed": (synth.ZED, 1920, 1080)}


def _f32(x):
    return np.ascontiguousarray(x, np.float32)


def _ulps(x, k):
    """x moved by k float32 ulps (k < 0: downwards), elementwise."""
    x = _f32(x).copy()
    toward = np.float32(np.inf) if k > 0 else np.float32(-np.inf)
    for _ in range(abs(k)):
        x = np.nextafter(x, toward)
    return x


def family(name, cal, seed=0):
    """(a, b): n x 2 float32 left / right points of one disparity family at the calibration `cal`."""
    c, w, h = CALS[cal]
    rng = np.random.default_rng(seed)
    n = 400
    a = _f32(np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], 1))
    a[:8] = [[0, 0], [w - 1, h - 1], [c["cx"], c["cy"]], [0.5, 0.5], [w / 2, 0], [0, h / 2], [1, 1], [w - 1, 0]]
    b = a.copy()
    if name == "zero":
        pass
    elif name == "ulps":                                # +-1..4 ulps of xl, y identical
        k = np.tile(np.array([1, 2, 3, 4, -1, -2, -3, -4]), n // 8)
        for s in np.unique(k):
            b[k == s, 0] = _ulps(a[k == s, 0], int(s))
    elif name == "subpixel":                            # 1e-3 .. 0.5 px, log-uniform
        b[:, 0] = a[:, 0] - _f32(np.exp(rng.uniform(np.log(1e-3), np.log(0.5), n)))
    elif name == "negative":                            # right point to the right of the left one: behind the rig
        b[:, 0] = a[:, 0] + _f32(np.exp(rng.uniform(np.log(1e-3), np.log(80.0), n)))
    elif name == "vertical":                            # zero horizontal disparity, a vertical mismatch
        b[:, 1] = a[:, 1] + _f32(rng.choice([-1, 1], n) * np.exp(rng.uniform(np.log(1e-4), np.log(3.0), n)))
    elif name == "outside":                             # outside the image and at +-1e5 px, ordinary disparities
        a = _f32(np.stack([rng.uniform(-3 * w, 4 * w, n), rng.uniform(-3 * h, 4 * h, n)], 1))
        a[:8] = [[1e5, 1e5], [-1e5, -1e5], [1e5, -1e5], [-1e5, 1e5], [1e5, c["cy"]], [c["cx"], -1e5], [-1e5, 0], [0, 1e5]]
        b = a.copy()
        b[:, 0] -= _f32(rng.uniform(0.5, 80, n))
        b[8:16, 0] = a[8:16, 0]                         # ... and a few at zero disparity
    else:
        raise ValueError(name)
    return a, _f32(b)


def threshold_family(cal, max_steps=48):
    """Disparities straddling |w| = FLT_EPSILON: for left points spread over the image (and its left part, where ulps
    are finest), step xr down from xl one ulp at a time and keep the steps whose cv2 w lies within a factor 4 of it."""
    c, w, h = CALS[cal]
    P_l, P_r = synth.proj_matrices(c)
    rng = np.random.default_rng(7)
    xs = np.concatenate([rng.uniform(1, 64, 40), rng.uniform(64, w, 40)])
    a = _f32(np.stack([xs, rng.uniform(0, h, len(xs))], 1))
    A, B = [a], [a.copy()]
    b = a.copy()
    for _ in range(max_steps):
        b = b.copy(); b[:, 0] = _ulps(b[:, 0], -1)
        A.append(a); B.append(b)
    a, b = np.concatenate(A), np.concatenate(B)
    wv = np.abs(cv2.triangulatePoints(P_l, P_r, a.T.copy(), b.T.copy())[3])
    keep = (wv > EPS / 4) & (wv < 4 * EPS)
    return a[keep], b[keep]


FAMILIES = ["zero", "ulps", "threshold", "subpixel", "negative", "vertical", "outside", "single"]


def points(name, cal):
    if name == "threshold":
        return threshold_family(cal)
    if name == "single":                                # n = 1, at zero disparity, away from the principal point
        a, b = family("zero", cal)
        return a[10:11].copy(), b[10:11].copy()
    return family(name, cal)


def cv2_triangulate(P_l, P_r, a, b):
    """The reference's two calls (src/main.cpp:170-171): (n x 4 homogeneous rows, n x 3 points)."""
    X4 = cv2.triangulatePoints(P_l, P_r, a.T.copy(), b.T.copy())
    return X4.T.copy(), cv2.convertPointsFromHomogeneous(X4.T.copy()).reshape(-1, 3)


def null_vector_f64(P_l, P_r, a, b):
    """Independent float64 restatement of the DLT: the right singular vector of the smallest singular value of the 4 x 4
    system (np.linalg.svd, LAPACK), unit norm."""
    Pl, Pr = P_l.astype(np.float64), P_r.astype(np.float64)
    out = np.zeros((len(a), 4))
    for i, ((x, y), (x2, y2)) in enumerate(zip(a.astype(np.float64), b.astype(np.float64))):
        A = np.array([x * Pl[2] - Pl[0], y * Pl[2] - Pl[1], x2 * Pr[2] - Pr[0], y2 * Pr[2] - Pr[1]])
        out[i] = np.linalg.svd(A)[2][3]
    return out


def rectified_geometry(P_l, P_r, a, b):
    """The exact rectified stereo point of float inputs with yl == yr: Z = -P_r[0,3] / d, d = xl - xr (in float64)."""
    Pl, Pr = P_l.astype(np.float64), P_r.astype(np.float64)
    x, y, xr = a[:, 0].astype(np.float64), a[:, 1].astype(np.float64), b[:, 0].astype(np.float64)
    Z = -Pr[0, 3] / (x - xr)
    return np.stack([(x - Pl[0, 2]) * Z / Pl[0, 0], (y - Pl[1, 2]) * Z / Pl[1, 1], Z], 1)


@pytest.fixture(scope="module")
def hostcheck(built):
    from visual_odom_b200 import build
    L = C.CDLL(build.build_hostcheck())
    p = lambda x: x.ctypes.data_as(C.c_void_p)

    def run(P_l, P_r, a, b):
        n = len(a)
        X, X4 = np.zeros((n, 3), np.float32), np.zeros((n, 4), np.float32)
        L.vo_hostcheck_triangulate4(p(_f32(P_l)), p(_f32(P_r)), p(_f32(a)), p(_f32(b)), n, p(X), p(X4))
        X3 = np.full((n, 3), np.nan, np.float32)
        L.vo_hostcheck_triangulate(p(_f32(P_l)), p(_f32(P_r)), p(_f32(a)), p(_f32(b)), n, p(X3))
        assert np.array_equal(X3, X)                    # the optional homogeneous output changes nothing
        return X4, X
    return run


def test_dehomogenize_threshold_is_cv2s():
    """convertPointsFromHomogeneous's rule on its own: divide only where |w| > FLT_EPSILON, strictly; NaN keeps 1."""
    up = np.nextafter(EPS, np.float32(1))
    ws = _f32([EPS, -EPS, up, -up, 0.0, -0.0, 1e-30, 1e-45, np.nan, np.nextafter(EPS, np.float32(0)), 1.0, -3e-5, 2e-7])
    X4 = _f32(np.stack([np.full(len(ws), 1.0), np.full(len(ws), 2.0), np.full(len(ws), 3.0), ws], 1))
    want = cv2.convertPointsFromHomogeneous(X4).reshape(-1, 3)
    got = P.dehomogenize_f32(X4)
    assert np.array_equal(got, want)
    assert np.array_equal(got[[0, 1, 4, 5, 6, 7, 8, 9]], np.tile(_f32([1, 2, 3]), (8, 1)))
    assert np.abs(got[2]).max() > 1e6


def _edge_asserts(name, H, X):
    """What each family is there for, so that it cannot pass vacuously."""
    w = np.abs(H[:, 3])
    if name in ("zero", "single"):
        assert np.all(w <= EPS)
        assert np.array_equal(X, H[:, :3])              # scale 1: the unit-norm column, within 1 m of the camera
    if name in ("ulps", "threshold"):
        assert (w <= EPS).sum() >= 10 and (w > EPS).sum() >= 10, "both sides of FLT_EPSILON occur"
        # one ulp more disparity moves the point from within 1 m of the camera to beyond 100 km
        assert np.abs(X[w > EPS, 2]).min() > 1e5 and np.abs(X[w <= EPS]).max() <= 1.0


@pytest.mark.parametrize("cal", sorted(CALS))
@pytest.mark.parametrize("name", FAMILIES)
def test_oracle_bit_exact_with_cv2(name, cal):
    P_l, P_r = synth.proj_matrices(CALS[cal][0])
    a, b = points(name, cal)
    H, X = cv2_triangulate(P_l, P_r, a, b)
    assert np.array_equal(P.triangulate(P_l, P_r, a, b), X)
    _edge_asserts(name, H, X)


@pytest.mark.parametrize("cal", sorted(CALS))
@pytest.mark.parametrize("name", FAMILIES)
def test_host_compiled_kernel_math_bit_exact_with_cv2(hostcheck, name, cal):
    P_l, P_r = synth.proj_matrices(CALS[cal][0])
    a, b = points(name, cal)
    H, X = cv2_triangulate(P_l, P_r, a, b)
    H_host, X_host = hostcheck(P_l, P_r, a, b)
    assert np.array_equal(H_host, H), "homogeneous column"
    assert np.array_equal(X_host, X), "3-D point"
    _edge_asserts(name, H_host, X_host)


@pytest.mark.parametrize("cal", sorted(CALS))
@pytest.mark.parametrize("name", FAMILIES)
def test_against_float64_null_vector_and_rectified_geometry(hostcheck, name, cal):
    c = CALS[cal][0]
    P_l, P_r = synth.proj_matrices(c)
    a, b = points(name, cal)
    H, X = hostcheck(P_l, P_r, a, b)
    ref = null_vector_f64(P_l, P_r, a, b)
    sign = np.where(np.sum(ref * H, 1) < 0, -1.0, 1.0)
    assert np.abs(H - sign[:, None] * ref).max() <= 6e-8, "homogeneous column vs the float64 null vector"
    rect = (a[:, 1] == b[:, 1]) & (a[:, 0] != b[:, 0]) & (np.abs(H[:, 3]) > EPS)
    if name in ("ulps", "threshold", "subpixel", "negative", "outside"):
        assert rect.sum() >= 10
    if rect.any():
        g = rectified_geometry(P_l, P_r, a[rect], b[rect])
        rel = np.linalg.norm(X[rect] - g, axis=1) / np.linalg.norm(g, axis=1)
        assert rel.max() <= 4e-7, "3-D point vs the exact rectified geometry"


@pytest.mark.parametrize("cal", sorted(CALS))
def test_oracle_triangulation_across_dense_disparities(hostcheck, cal):
    """A broad sweep, 1e-3 .. 200 px of either sign with sub-pixel vertical noise, for the float64 bounds above."""
    c, w, h = CALS[cal]
    P_l, P_r = synth.proj_matrices(c)
    rng = np.random.default_rng(11)
    n = 4000
    a = _f32(np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], 1))
    d = rng.choice([-1, 1], n) * np.exp(rng.uniform(np.log(1e-3), np.log(200.0), n))
    b = a.copy(); b[:, 0] = _f32(a[:, 0] - d)
    H, X = hostcheck(P_l, P_r, a, b)
    Hc, Xc = cv2_triangulate(P_l, P_r, a, b)
    assert np.array_equal(H, Hc) and np.array_equal(X, Xc)
    ref = null_vector_f64(P_l, P_r, a, b)
    sign = np.where(np.sum(ref * H, 1) < 0, -1.0, 1.0)
    assert np.abs(H - sign[:, None] * ref).max() <= 6e-8
    g = rectified_geometry(P_l, P_r, a, b)
    ok = np.abs(H[:, 3]) > EPS
    assert ok.all()
    assert (np.linalg.norm(X - g, axis=1) / np.linalg.norm(g, axis=1)).max() <= 4e-7


def test_sky_option_keeps_the_rest_of_the_scene():
    """The band replaces only its own pixels: below it the images, noise included, are those of the default scene, and
    the left / right images of one time are identical inside it."""
    u0 = synth.stereo_unit(640, 240, 3)
    u = synth.stereo_unit(640, 240, 3, sky=0.35)
    for k in ("l0", "r0", "l1", "r1"):
        assert np.array_equal(u[k][120:], u0[k][120:]), k
    assert np.array_equal(u["l0"][:80], u["r0"][:80]) and np.array_equal(u["l1"][:70], u["r1"][:70])
    assert not np.array_equal(u["l0"][:80], u["l1"][:80])
