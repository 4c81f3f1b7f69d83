"""The run-time LK, validity-filter and PnP parameters of vo_params away from the reference's literals: the oracle
(oracle/lk_ref.c, oracle/pnp_ref.py and the parameterised glue of oracle/ref_path.py) against cv2 4.13.0, bit for bit,
and the parameters vo_create refuses.

Where cv2 does not simply take a parameter as given, the oracle (and the library) do what cv2 does:
- calcOpticalFlowPyrLK clamps maxCount to [0, 100], as it clamps epsilon to [0, 10];
- LKTrackerInvoker keeps minEigThreshold as a float and compares minEig with it in float, so a threshold that rounds to
  a window's minEig keeps the window;
- a window whose normal matrix has D < FLT_EPSILON is rejected even at minEigThreshold 0 (flat and saturated patches);
- solvePnPRansac runs at least one RANSAC iteration for any iterationsCount, and from six points on asserts
  0 < confidence < 1.

The fixtures here (images, starts, PnP sets) are shared with tests/test_gpu_params.py."""
import functools
import math

import numpy as np
import pytest

from visual_odom_b200 import synth

cv2 = pytest.importorskip("cv2")

FLT_EPSILON = np.float32(1.1920928955078125e-07)
LK_ITERS = (-3, 0, 1, 2, 7, 100, 101, 150)
LK_MIN_EIGS = (0.0, 1e-4, 5e-3, 0.02)
CIRC_THRESHOLDS = (-1, 1, 2, 5)


# ----------------------------------------------------------------------------- images and starts
def multiscale_pair(w, h, seed, shift=(9.3, -5.6)):
    """Two views of one texture with detail at 4 to 1024 pixel scales (so that every level of an 8-image pyramid sees
    structure), the second shifted by `shift` pixels, each with its own N(0, 1) sensor noise."""
    rng = np.random.default_rng(seed)
    m = 64
    W, H = w + 2 * m, h + 2 * m
    acc = np.zeros((H, W), np.float64)
    for cell in (4, 16, 64, 256, 1024):
        lo = rng.normal(0, 1, (H // cell + 3, W // cell + 3))
        acc += 40.0 * cv2.resize(lo, (W + 2 * cell, H + 2 * cell), interpolation=cv2.INTER_CUBIC)[cell:cell + H, cell:cell + W]
    T = np.clip(128 + acc, 0, 255).astype(np.float32)
    views = []
    for dx, dy in ((0.0, 0.0), shift):
        views.append(cv2.warpAffine(T, np.float32([[1, 0, m + dx], [0, 1, m + dy]]), (w, h), flags=cv2.INTER_LINEAR))
    noise = rng.normal(0, 1, (2, h, w))
    return [np.clip(np.rint(v + n), 0, 255).astype(np.uint8) for v, n in zip(views, noise)]


def starts(w, h, n, seed, border=30):
    """n starts scattered over the image and `border` pixels around it (some leave the image at coarse or fine levels)."""
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(-border, w + border, n), rng.uniform(-border, h + border, n)], 1).astype(np.float32)


# name -> (w, h, pyramid images at max_level 7): 2816 x 2816 reaches VO_MAX_LEVELS = 8 images, 1241 x 376 stops at 5
# (its level 5 would be 39 x 12), 320 x 160 at 3 (level 3 would be 40 x 20)
LK_IMAGES = {"deep": (2816, 2816, 8), "kitti": (1241, 376, 5), "small": (320, 160, 3)}


@functools.lru_cache(maxsize=None)
def lk_image(name):
    """(prev, next, starts) of one LK_IMAGES entry."""
    w, h, _ = LK_IMAGES[name]
    if name == "small":
        u = synth.stereo_unit(w, h, 5)
        prev, nxt = u["l0"], u["r0"]
    else:
        prev, nxt = multiscale_pair(w, h, 3 if name == "deep" else 4)
    return prev, nxt, starts(w, h, 400, 17)


@functools.lru_cache(maxsize=None)
def flat_pair():
    """320 x 160 textured views with a flat (128), a black (0) and a saturated (255) block in both; starts at the block
    centres and half a window off them, and scattered ones."""
    u = synth.stereo_unit(320, 160, 6)
    prev, nxt = u["l0"].copy(), u["r0"].copy()
    blocks = [(20, 30, 128), (20, 130, 0), (90, 220, 255)]       # (y0, x0, value), 60 x 60 each
    for img in (prev, nxt):
        for y0, x0, v in blocks:
            img[y0:y0 + 60, x0:x0 + 60] = v
    pts = []
    for y0, x0, _ in blocks:
        for dy in (-25.5, -10, 0, 0.25, 10, 25):
            for dx in (-25, -10.5, 0, 0.75, 10, 25):
                pts.append((x0 + 30 + dx, y0 + 30 + dy))
    pts = np.concatenate([np.array(pts, np.float32), starts(320, 160, 100, 23)])
    return prev, nxt, pts


def lk_both(prev, nxt, pts, **kw):
    """(cv2 (out, status, err), oracle (out, status, err, log)) of one call with the LK keywords of ref_path."""
    from oracle import cref, ref_path
    ref = ref_path.lk_cv2(prev, nxt, pts, with_err=True, **kw)
    got = cref.lk_track(prev, nxt, pts, max_level=kw.get("max_level", 3), max_count=kw.get("max_iters", 30),
                        epsilon=kw.get("epsilon", 0.01), min_eig=kw.get("min_eig", 1e-3), return_log=True)
    return ref, got


def assert_lk_equal(ref, got, where):
    o, s, e = ref
    go, gs, ge = got[:3]
    assert np.array_equal(gs, s), f"{where}: status differs at {np.nonzero(gs != s)[0][:8]}"
    bad = np.nonzero((go != o).any(1))[0]
    assert len(bad) == 0, f"{where}: positions differ at {len(bad)} points, first {bad[:8]}"
    assert np.array_equal(ge[s == 1], e[s == 1]), f"{where}: err differs"


def logged_thresholds(n=200):
    """Thresholds T within a quarter ulp of a level-0 minEig f of the small pair's starts (float(T) == f), on both sides,
    with the starts they belong to: [(start, T_above, T_below)].  cv2 keeps such a window (f < f is false); a comparison
    in double would drop it at T_above."""
    from oracle import cref
    prev, nxt, pts = lk_image("small")
    _, _, _, log = cref.lk_track(prev, nxt, pts, min_eig=0.0, return_log=True)
    st = log[((log["kind"] == cref.EV_SETUP) | (log["kind"] == cref.EV_REJECT)) & (log["level"] == 0)]
    st = st[(st["min_eig"] > 0) & (st["D"] >= FLT_EPSILON)]
    assert len(st) >= n
    out = []
    for e in st[:n]:
        f = np.float32(e["min_eig"])
        up = float(np.nextafter(f, np.float32(1))) - float(f)
        down = float(f) - float(np.nextafter(f, np.float32(0)))
        t_above, t_below = float(f) + up / 4, float(f) - down / 4
        assert np.float32(t_above) == f and np.float32(t_below) == f and t_above > float(f) > t_below
        out.append((pts[e["pt"]], t_above, t_below))
    return out


# ----------------------------------------------------------------------------- LK
@pytest.mark.parametrize("name", list(LK_IMAGES))
@pytest.mark.parametrize("max_level", range(8))
def test_lk_max_level(built, name, max_level):
    """Every pyramid depth the library accepts, on images that reach it and on images that stop short of it."""
    from oracle import cref
    prev, nxt, pts = lk_image(name)
    ref, got = lk_both(prev, nxt, pts, max_level=max_level)
    assert_lk_equal(ref, got, f"{name} max_level={max_level}")
    nlev = min(max_level + 1, LK_IMAGES[name][2])
    assert cref.Pyramid(prev, max_level=max_level).nlevels() == nlev
    log = got[3]
    setups = log[log["kind"] == cref.EV_SETUP]
    assert (setups["level"] == nlev - 1).sum() > 50, "the coarsest level solves few windows"
    assert 0.5 * len(pts) < ref[1].sum() < len(pts)


@pytest.mark.parametrize("max_iters", LK_ITERS)
def test_lk_max_iters(built, max_iters):
    """maxCount outside [0, 100] is clamped: -3 runs as 0, 101 and 150 as 100.  epsilon = 0 lets the count end every
    solve that the half-step exit does not."""
    prev, nxt, pts = lk_image("small")
    ref, got = lk_both(prev, nxt, pts, max_iters=max_iters, epsilon=0.0)
    assert_lk_equal(ref, got, f"max_iters={max_iters}")
    clamped = min(max(max_iters, 0), 100)
    if clamped != max_iters:
        ref_c, _ = lk_both(prev, nxt, pts, max_iters=clamped, epsilon=0.0)
        assert_lk_equal(ref_c, got, f"max_iters={max_iters} against {clamped}")
    if max_iters == 150:
        from oracle import cref
        cap = got[3][got[3]["kind"] == cref.EV_CAP]
        assert len(cap) > 0 and cap["iter"].max() == 99        # the clamp decides: solves run into the 100-iteration cap


@pytest.mark.parametrize("min_eig", LK_MIN_EIGS)
@pytest.mark.parametrize("name", ["small", "kitti"])
def test_lk_min_eig(built, name, min_eig):
    from oracle import cref
    prev, nxt, pts = lk_image(name)
    ref, got = lk_both(prev, nxt, pts, min_eig=min_eig)
    assert_lk_equal(ref, got, f"{name} min_eig={min_eig}")
    if min_eig > 0:
        rej = got[3][got[3]["kind"] == cref.EV_REJECT]
        assert (rej["min_eig"] < np.float32(min_eig)).any()


@pytest.mark.parametrize("side", ["above", "below"])
def test_lk_min_eig_threshold_rounding_to_a_windows_min_eig(built, side):
    """Thresholds taken from the event log, a quarter ulp above or below a level-0 minEig: cv2 compares in float, keeps
    the window on both sides, and the oracle must do the same (one start per call, each at its own threshold)."""
    from oracle import cref, ref_path
    prev, nxt, _ = lk_image("small")
    pp, npy = cref.Pyramid(prev, 21, 3, True), cref.Pyramid(nxt, 21, 3, False)
    kept = 0
    for p, t_above, t_below in logged_thresholds():
        t = t_above if side == "above" else t_below
        p = p.reshape(1, 2)
        ref = ref_path.lk_cv2(prev, nxt, p, min_eig=t, with_err=True)
        got = cref.lk_track(prev, nxt, p, min_eig=t, prev_pyr=pp, next_pyr=npy)
        assert_lk_equal(ref, got, f"start {p.ravel()} threshold {t!r}")
        kept += int(ref[1][0])
    assert kept >= 150                  # most windows are kept (a few starts end outside the image)


def test_flat_and_saturated_windows_take_the_determinant_rejection(built):
    """At minEigThreshold 0 a flat, black or saturated window passes the minEig test (0 < 0 is false) and is rejected by
    D < FLT_EPSILON, at every level; cv2 and the oracle agree on every start, and the log shows the branch was taken."""
    from oracle import cref
    prev, nxt, pts = flat_pair()
    ref, got = lk_both(prev, nxt, pts, min_eig=0.0)
    assert_lk_equal(ref, got, "flat blocks")
    log = got[3]
    rej = log[log["kind"] == cref.EV_REJECT]
    by_d = rej[(rej["min_eig"] >= 0) & (rej["D"] < FLT_EPSILON)]
    assert (by_d["level"] == 0).sum() >= 12 and len(np.unique(by_d["level"])) >= 2
    assert (ref[1][np.unique(by_d["pt"][by_d["level"] == 0])] == 0).all()
    # at the default threshold the same windows are rejected by minEig < 0.001 before D is looked at
    ref_d, got_d = lk_both(prev, nxt, pts)
    assert_lk_equal(ref_d, got_d, "flat blocks, default threshold")


# ----------------------------------------------------------------------------- checkValidMatch
def _reference_check_valid_match(points, points_return, threshold):
    """visualOdometry.cpp:44-61 element by element: float differences, std::max of std::abs, assigned to an int."""
    out = []
    for p, q in zip(points, points_return):
        d = max(abs(np.float32(p[0]) - np.float32(q[0])), abs(np.float32(p[1]) - np.float32(q[1])))
        offset = int(d)                                  # float -> int truncates toward zero
        out.append(not (offset > threshold))
    return np.array(out, bool)


def circ_pairs():
    """Point pairs whose max-abs difference sits on and around the integers 0 .. 7, in x or in y, with either sign."""
    rng = np.random.default_rng(8)
    d = np.concatenate([np.arange(8, dtype=np.float32), np.arange(8, dtype=np.float32) - np.float32(1e-3),
                        np.arange(8, dtype=np.float32) + np.float32(1e-3), rng.uniform(0, 8, 200).astype(np.float32)])
    d = np.concatenate([d, -d])
    p = rng.uniform(0, 1000, (len(d), 2)).astype(np.float32)
    q = p.copy()
    axis = np.arange(len(d)) % 2
    q[np.arange(len(d)), axis] += d
    q[np.arange(len(d)), 1 - axis] += (d * np.float32(0.5)).astype(np.float32)
    return p, q


@pytest.mark.parametrize("threshold", CIRC_THRESHOLDS + (0,))
def test_check_valid_match_thresholds(threshold):
    from oracle import ref_path
    p, q = circ_pairs()
    got = ref_path.check_valid_match(p, q, threshold)
    want = _reference_check_valid_match(p, q, threshold)
    assert np.array_equal(got, want)
    if threshold >= 0:
        assert 0 < got.sum() < len(got)
    else:
        assert not got.any()                 # no offset is below 0


# ----------------------------------------------------------------------------- solvePnPRansac
PNP_SETS = {"s300": (300, 0.1, 0.2, 4), "s1500": (1500, 0.15, 0.3, 1), "s40": (40, 0.3, 0.4, 9)}
PNP_ITERS = (-5, 0, 1, 3, 31, 32, 33, 2000)
PNP_REPROJ = (0.1, 0.5, 2.0, -1.0, 0.0)
PNP_CONF = (0.5, 0.99)
T_PREV = np.array([0.02, 0.0, -0.8])


@functools.lru_cache(maxsize=None)
def pnp_set(name):
    X, x, K, _ = synth.pnp_stress_set(*PNP_SETS[name][:3], seed=PNP_SETS[name][3])
    return X, x, K


def cv2_pnp(X, x, K, iterations, reproj, confidence):
    ok, rv, tv, inl = cv2.solvePnPRansac(X.reshape(-1, 1, 3), x.reshape(-1, 1, 2), K, np.zeros(4), np.zeros(3), T_PREV.copy(),
                                         True, iterations, reproj, confidence, None, cv2.SOLVEPNP_ITERATIVE)
    inl = np.zeros(0, np.int32) if inl is None else inl.ravel().astype(np.int32)
    return ok, rv.ravel(), tv.ravel(), inl


@pytest.mark.parametrize("iterations", PNP_ITERS)
@pytest.mark.parametrize("name", list(PNP_SETS))
def test_pnp_iterations_reprojection_and_confidence(name, iterations):
    from oracle import pnp_ref
    X, x, K = pnp_set(name)
    for reproj in PNP_REPROJ:
        if iterations == 2000 and reproj in (0.0, 0.1):
            continue                     # no early stop: thousands of pure-Python RANSAC iterations
        for conf in PNP_CONF:
            where = f"{name} iterations={iterations} reproj={reproj} confidence={conf}"
            ok, rv, tv, inl = cv2_pnp(X, x, K, iterations, reproj, conf)
            res = pnp_ref.solve_pnp_ransac(X, x, K, np.zeros(3), T_PREV, iterations=iterations, reproj=reproj, confidence=conf)
            assert res["ok"] == ok, where
            assert np.array_equal(res["inliers"], inl), f"{where}: {len(res['inliers'])} inliers, cv2 {len(inl)}"
            assert res["iters"] >= 1, where
            if ok:
                assert np.linalg.norm(res["rvec"] - rv) <= 1e-6 * max(1.0, np.linalg.norm(rv)), where
                assert np.linalg.norm(res["tvec"] - tv) <= 1e-6 * np.linalg.norm(tv), where
    if iterations <= 0:                  # one iteration, as at iterationsCount 1
        for conf in PNP_CONF:
            a = pnp_ref.solve_pnp_ransac(X, x, K, np.zeros(3), T_PREV, iterations=iterations, confidence=conf)
            b = pnp_ref.solve_pnp_ransac(X, x, K, np.zeros(3), T_PREV, iterations=1, confidence=conf)
            assert a["iters"] == b["iters"] == 1 and np.array_equal(a["inliers"], b["inliers"])
        if name == "s300":
            assert len(a["inliers"]) == 77


@pytest.mark.parametrize("confidence", [0.0, 1.0, -0.1, 1.5, math.nan])
def test_pnp_confidence_outside_the_unit_interval(confidence):
    """cv2 asserts 0 < confidence < 1 once RANSAC runs (six points or more) and the oracle refuses the same; five points
    (no RANSAC) are solved as at any confidence."""
    from oracle import pnp_ref
    X, x, K = pnp_set("s300")
    for n in (6, 300):
        with pytest.raises(cv2.error):
            cv2_pnp(X[:n], x[:n], K, 100, 0.5, confidence)
        with pytest.raises(ValueError, match="confidence"):
            pnp_ref.solve_pnp_ransac(X[:n], x[:n], K, np.zeros(3), T_PREV, iterations=100, confidence=confidence)
    ok, rv, tv, inl = cv2_pnp(X[:5], x[:5], K, 100, 0.5, confidence)
    res = pnp_ref.solve_pnp_ransac(X[:5], x[:5], K, np.zeros(3), T_PREV, iterations=100, confidence=confidence)
    assert ok and res["ok"] and np.array_equal(res["inliers"], inl)
    assert np.array_equal(res["rvec"], rv) and np.array_equal(res["tvec"], tv)


# ----------------------------------------------------------------------------- vo_create
@pytest.mark.parametrize("field,value", [("pnp_confidence", 0.0), ("pnp_confidence", 1.0), ("pnp_confidence", -0.1),
                                         ("pnp_confidence", math.nan), ("pnp_confidence", 1.5),
                                         ("max_features", 0), ("max_features", -4)])
def test_vo_create_refuses(built, field, value):
    """Checked before the device query (as fast_threshold is), so the refusal is the same with and without a GPU."""
    from visual_odom_b200.capi import VO_E_INVALID, Context, VoError
    with pytest.raises(VoError) as e:
        Context(0, **{field: value})
    assert e.value.code == VO_E_INVALID and field in str(e.value), str(e.value)
