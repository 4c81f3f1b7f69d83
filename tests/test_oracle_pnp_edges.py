"""The pose tail at its edges: oracle/pnp_ref.py (and, where it applies, the kernels' own math compiled for the host)
against cv2 4.13.0's solvePnPRansac, called as the reference calls it (src/visualOdometry.cpp:176-178).

- n == 5 (= the model size): OpenCV runs no RANSAC but one EPnP on all five points, unrefined, all five inliers.
- n = 6 .. 16: the subset draw redraws on duplicates most often here, so any drift of the RNG stream shows.
- The mono branch at n == 5: findEssentialMat returns every five-point candidate stacked, recoverPose refuses a stack.
- Fixture sets, built here and imported by tests/test_gpu_pnp_edges.py.  Each builder asserts, when it builds a set, the
  property the set exists for, against the oracle and cv2:
    wave sets        the final adaptive iteration count inside / on the edges of the kernels' waves [0,32) [32,128) [128,500)
    degenerate sets  no model, 5x duplicated correspondences (ties: the first best wins), a planar scene, points behind
                     the camera, points as far as Z = 1e30
    threshold set    points moved so that their squared f32 error is 0.25f or one ulp either side of it
"""
import ctypes as C
import functools

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from oracle import essential_ref as er  # noqa: E402
from oracle import pnp_ref as P  # noqa: E402
from visual_odom_b200 import synth  # noqa: E402

T_PREV = np.array([0.02, 0.0, -0.8])
CONF = float(np.float32(0.999))              # `float confidence = 0.999` (visualOdometry.cpp:170)
THR = np.float32(0.25)                       # (float)(0.5 * 0.5)
WAVES = (0, 32, 128, 500)                    # the kernels' RANSAC waves (pnp.cu vo_launch_pnp)


def cv2_pnp(X, x, K, t_prev=T_PREV):
    """cv::solvePnPRansac exactly as the reference calls it -> (ok, rvec, tvec, inliers)."""
    ok, rv, tv, inl = cv2.solvePnPRansac(
        np.ascontiguousarray(X, np.float32).reshape(-1, 1, 3), np.ascontiguousarray(x, np.float32).reshape(-1, 1, 2),
        np.asarray(K, np.float32), np.zeros((4, 1)), np.zeros((3, 1)), np.asarray(t_prev, np.float64).reshape(3, 1).copy(),
        True, 500, 0.5, CONF, None, cv2.SOLVEPNP_ITERATIVE)
    inl = np.zeros(0, np.int32) if inl is None else inl.ravel().astype(np.int32)
    return bool(ok), rv.ravel(), tv.ravel(), inl


def oracle_pnp(X, x, K, t_prev=T_PREV):
    return P.solve_pnp_ransac(X, x, K, np.zeros(3), t_prev, confidence=CONF)


def replay(X, x, K):
    """The RANSAC stream of solvePnPRansac run past its stop to the end of the wave the GPU computes: the kernels
    evaluate every iteration of a wave below the bound the wave started with, and the replay must ignore those past
    the bound.  Returns dict(iters = iterations run, best_it, max_good, counts[it] for every computed iteration,
    late_better = computed iterations at or past `iters` whose count beats the final best, ties = iterations before the
    stop with another inlier set of the same size as the best so far, which must not replace it)."""
    X = np.asarray(X, np.float32); x = np.asarray(x, np.float32)
    K64 = np.asarray(K, np.float32).astype(np.float64)
    n = len(X)
    rng = P.CvRNG()
    niters, max_good, best_it, it = 500, 0, -1, 0
    counts, masks, ties = [], [], []
    w = 0
    while True:
        it1 = WAVES[w + 1]
        last = min(it1, niters)                              # what this wave computes
        for j in range(len(counts), last):
            idx = P.ransac_subset(rng, n, 5)
            rv, tv = P.epnp(X[idx], x[idx], K64)
            masks.append(P.reproj_err_f32(X, x, rv, tv, K64) <= THR)
            counts.append(int(masks[-1].sum()))
        while it < it1 and it < niters:
            if counts[it] > max(max_good, 4):
                best_it, max_good = it, counts[it]
                niters = P.ransac_update_num_iters(CONF, float(n - max_good) / n, 5, niters)
            elif counts[it] == max_good > 4 and not np.array_equal(masks[it], masks[best_it]):
                ties.append(it)
            it += 1
        if it >= niters or it1 >= 500:
            break
        w += 1
    late = [j for j in range(it, len(counts)) if counts[j] > max_good]
    return dict(iters=it, best_it=best_it, max_good=max_good, counts=counts, late_better=late, ties=ties)


def check_against_cv2(X, x, K, t_prev=T_PREV, pose_tol=1e-6):
    """oracle == cv2 on one set: success flag, inlier list, pose within pose_tol; returns the oracle's result."""
    ok, rv, tv, inl = cv2_pnp(X, x, K, t_prev)
    res = oracle_pnp(X, x, K, t_prev)
    assert res["ok"] == ok
    assert np.array_equal(res["inliers"], inl)
    if ok:
        assert np.abs(res["rvec"] - rv).max() <= pose_tol * max(1.0, np.abs(rv).max())
        assert np.abs(res["tvec"] - tv).max() <= pose_tol * max(1.0, np.abs(tv).max())
    else:
        assert res["iters"] == 500
    return res


# ----------------------------------------------------------------------------- fixture builders
def _stress(n, sigma, outl, seed):
    X, x, K, _ = synth.pnp_stress_set(n, sigma, outl, seed=seed)
    return X, x, K


# (n, sigma, outlier fraction, seed) found by a seed search; the builder asserts what each one is for.  No seed of that
# search (8 noise / outlier mixes x 10 seeds) stopped exactly on 32 or 128 iterations.
WAVE_SPECS = {
    "below_32": ((300, 0.1, 0.2, 0), lambda r: 0 < r["iters"] < 32),
    "between_32_128": ((300, 0.1, 0.3, 0), lambda r: 32 < r["iters"] < 128),
    "between_128_500": ((300, 0.2, 0.5, 2), lambda r: 128 < r["iters"] < 500),
    "stays_500": ((600, 0.1, 0.88, 0), lambda r: r["iters"] == 500 and r["best_it"] >= 0),
    "late_better": ((300, 0.1, 0.1, 0), lambda r: len(r["late_better"]) > 0),
}


@functools.lru_cache(maxsize=None)
def wave_set(name):
    """A stress set whose adaptive iteration count is `name`; returns (X, x, K, oracle result, replay)."""
    (n, sigma, outl, seed), prop = WAVE_SPECS[name]
    X, x, K = _stress(n, sigma, outl, seed)
    r = replay(X, x, K)
    assert prop(r), (name, r["iters"], r["best_it"], r["late_better"])
    res = check_against_cv2(X, x, K)
    assert res["iters"] == r["iters"]
    return X, x, K, res, r


@functools.lru_cache(maxsize=None)
def degenerate_set(name):
    """Sets at the degenerate ends; returns (X, x, K, oracle result)."""
    rng = np.random.default_rng(7)
    K = synth.proj_matrices()[0][:, :3].copy()
    if name == "all_outliers":
        X = np.stack([rng.uniform(-30, 30, 200), rng.uniform(-3, 6, 200), rng.uniform(6, 80, 200)], 1).astype(np.float32)
        x = np.stack([rng.uniform(0, 1241, 200), rng.uniform(0, 376, 200)], 1).astype(np.float32)
    elif name == "dup5":
        X, x, K = _stress(60, 0.15, 0.3, 4)
        X = np.repeat(X, 5, 0); x = np.repeat(x, 5, 0)
    elif name == "planar":
        X, x, K = _plane_set(rng)
    elif name == "behind":
        X, x, K, _ = synth.pnp_stress_set(200, 0.1, 0.2, seed=8)
        X = X.copy()
        back = rng.random(len(X)) < 0.2
        X[back] *= np.float32(-1)                          # mirrored through the camera: same ray, negative depth
    elif name == "far":
        X, x, K, _ = synth.pnp_stress_set(200, 0.1, 0.2, seed=9)
        X = X.copy()
        far = np.arange(len(X)) % 7 == 3
        X[far] *= np.logspace(3, 28.5, int(far.sum()))[:, None].astype(np.float32)    # Z up to ~1e30: the ray is kept
    else:
        raise KeyError(name)
    X = np.ascontiguousarray(X, np.float32); x = np.ascontiguousarray(x, np.float32)
    res = check_against_cv2(X, x, K)
    if name == "all_outliers":
        assert not res["ok"]
    if name == "dup5":
        r = replay(X, x, K)
        # a later iteration with the final best count and another inlier set: only `count > best` keeps the first
        assert res["ok"] and any(t > r["best_it"] for t in r["ties"]), "no tie with another inlier set on the final best"
        assert res["iters"] == r["iters"]
    return X, x, K, res


def _plane_set(rng):
    """Every point on the ground plane Y = 1.65 (exactly, in f32)."""
    n = 200
    K = synth.proj_matrices()[0][:, :3].copy()
    X = np.stack([rng.uniform(-20, 20, n), np.full(n, 1.65), rng.uniform(6, 60, n)], 1).astype(np.float32)
    R = P.rodrigues(np.array(synth.EGO_RVEC, np.float64))
    Xc = X.astype(np.float64) @ R.T + np.asarray(synth.EGO_T, np.float64)
    x = np.stack([Xc[:, 0] / Xc[:, 2] * K[0, 0] + K[0, 2], Xc[:, 1] / Xc[:, 2] * K[1, 1] + K[1, 2]], 1)
    x += rng.normal(0, 0.15, x.shape)
    out = rng.random(n) < 0.3
    x[out] += rng.uniform(-15, 15, (int(out.sum()), 2))
    return X, x.astype(np.float32), K


DEGENERATE = ("all_outliers", "dup5", "planar", "behind", "far")


def _boundary_offsets(qx, qy, target, flip, sign):
    """(dx, dy), multiples of the grids qx, qy, whose unfused f32 dx*dx + dy*dy is `target`; `flip`: a fused
    fmaf(dx, dx, dy*dy) lands on the other side of 0.25f."""
    f32 = np.float32
    dx = (np.arange(int(0.2 / qx), int(0.45 / qx)) * qx).astype(f32)
    dx2 = dx * dx                                                    # f32 products, as the kernels round them
    rem = float(target) - dx2.astype(np.float64)
    dx, dx2, rem = dx[rem > 0], dx2[rem > 0], rem[rem > 0]
    m0 = (np.sqrt(rem) / qy).astype(np.int64)
    for d in range(-2, 3):
        dy = ((m0 + d) * qy).astype(f32)
        dy2 = dy * dy
        fused = (dx.astype(np.float64) ** 2 + dy2.astype(np.float64)).astype(f32)   # exact in double, one rounding
        hit = ((dx2 + dy2) == target) & (((fused <= THR) != (target <= THR)) == flip)
        if hit.any():
            j = int(np.argmax(hit))
            return f32(sign[0] * dx[j]), f32(sign[1] * dy[j])
    return None


@functools.lru_cache(maxsize=None)
def threshold_set():
    """A stress set where 48 points sit on the inlier threshold of the best model: their f32 squared error is 0.25f or one
    ulp either side, and for half of them a fused multiply-add would put them on the other side.  Returns
    (X, x, K, oracle result, moved indices, expected in-mask of the moved points)."""
    X, x, K = _stress(1000, 0.15, 0.3, 11)
    r0 = replay(X, x, K)
    res0 = oracle_pnp(X, x, K)
    rv, tv = res0["model"]
    K64 = np.asarray(K, np.float32).astype(np.float64)
    rng = P.CvRNG()
    subsets = [P.ransac_subset(rng, len(X), 5) for _ in range(r0["best_it"] + 1)]
    p = P.project_points(X, rv, tv, K64).astype(np.float32)
    gen = np.random.default_rng(3)
    cand = [i for i in gen.permutation(len(X)) if i not in subsets[-1] and np.all(np.abs(p[i]) < 2000)]
    targets = [np.nextafter(THR, np.float32(0)), THR, np.nextafter(THR, np.float32(1))]
    # a fused sum differs from the unfused one by at most one ulp, so it can only cross from 0.25f (up) or from one
    # ulp above (down): 16 and 8 cross, 8 at each of the three targets do not
    plan = [(THR, True)] * 16 + [(targets[2], True)] * 8 + [(t, False) for t in targets] * 8
    x = x.copy()
    moved, want = [], []
    for i in cand:
        if len(moved) == len(plan):
            break
        target, flip = plan[len(moved)]
        if flip and abs(p[i, 0]) >= 512:
            continue                                       # dx needs more bits than a coarser grid gives for dx*dx to round
        qx, qy = (float(np.spacing(np.float32(abs(v)) + np.float32(0.5))) for v in p[i])
        sign = (1 if gen.random() < 0.5 else -1, 1 if gen.random() < 0.5 else -1)
        off = _boundary_offsets(qx, qy, target, flip, sign)
        if off is None:
            continue
        u = np.float32(p[i, 0] + off[0]), np.float32(p[i, 1] + off[1])
        if np.float32(u[0] - p[i, 0]) != off[0] or np.float32(u[1] - p[i, 1]) != off[1]:
            continue                                       # p - u not exact in f32 here
        x[i] = u
        moved.append(i); want.append(bool(target <= THR))
    assert len(moved) == len(plan)
    moved = np.array(moved); want = np.array(want)
    err = P.reproj_err_f32(X[moved], x[moved], rv, tv, K64)
    assert set(err.tolist()) == {float(t) for t in targets}
    r = replay(X, x, K)
    assert r["best_it"] == r0["best_it"], "moving the points changed the best iteration"
    res = check_against_cv2(X, x, K)                       # cv2's mask = the unfused sum (what it is checked for)
    inl = set(res["inliers"].tolist())
    assert [i in inl for i in moved] == want.tolist()
    return X, x, K, res, moved, want


# ----------------------------------------------------------------------------- n == 5
def five_point_sets():
    """>= 200 five-point stress sets, sigma in [0, 0.5], outliers 0 .. 60 %."""
    for s in range(220):
        sigma = 0.05 * (s % 11)
        outl = 0.1 * (s % 7)
        yield _stress(5, sigma, outl, 1000 + s)


def _hostcheck():
    from visual_odom_b200 import build
    return C.CDLL(build.build_hostcheck())


def test_five_points_is_one_epnp_bit_for_bit(built):
    """n == 5: cv2 runs one EPnP on all five, no RANSAC, no LM; the oracle and the product's EPnP (host build) give the
    same rvec, tvec and inliers bit for bit."""
    L = _hostcheck()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    sets = 0
    for X, x, K in five_point_sets():
        ok, rv, tv, inl = cv2_pnp(X, x, K)
        res = oracle_pnp(X, x, K)
        assert ok and res["ok"] and res["iters"] == 0
        assert np.array_equal(inl, np.arange(5)) and np.array_equal(res["inliers"], inl)
        assert np.array_equal(res["rvec"], rv) and np.array_equal(res["tvec"], tv)
        rh = np.zeros(3); th = np.zeros(3); Rh = np.zeros(9)
        L.vo_hostcheck_epnp5(p(np.ascontiguousarray(X)), p(np.ascontiguousarray(x)),
                             p(np.ascontiguousarray(K, np.float32).ravel()), p(rh), p(th), p(Rh))
        assert np.array_equal(rh, rv) and np.array_equal(th, tv)
        assert np.array_equal(Rh.reshape(3, 3), cv2.Rodrigues(rv)[0])
        sets += 1
    assert sets >= 200


def identical_five():
    X, x, K = _stress(5, 0.1, 0.0, 19)
    return np.repeat(X[:1], 5, 0), np.repeat(x[:1], 5, 0), K


def test_five_identical_points_keep_cv2s_non_finite_pose(built):
    """Five identical correspondences: cv2 still reports success, rvec = 0 (its Rodrigues refuses a non-finite matrix)
    and tvec = nan.  The oracle and the product's math have the same finite components, with the same values."""
    X, x, K = identical_five()
    ok, rv, tv, inl = cv2_pnp(X, x, K)
    assert ok and np.array_equal(inl, np.arange(5))
    res = oracle_pnp(X, x, K)
    L = _hostcheck()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rh = np.zeros(3); th = np.zeros(3); Rh = np.zeros(9)
    L.vo_hostcheck_epnp5(p(X), p(x), p(np.ascontiguousarray(K, np.float32).ravel()), p(rh), p(th), p(Rh))
    for r_, t_ in ((res["rvec"], res["tvec"]), (rh, th)):
        for got, want in ((r_, rv), (t_, tv)):
            assert np.array_equal(np.isfinite(got), np.isfinite(want))
            assert np.array_equal(got[np.isfinite(want)], want[np.isfinite(want)])
    assert res["ok"] and np.array_equal(res["inliers"], np.arange(5))


@pytest.mark.parametrize("n", [6, 7, 8, 9, 10, 12, 16])
def test_small_counts_follow_cv2s_subset_stream(n):
    """n = 6 .. 16: inlier masks identical to cv2, pose within 1e-6."""
    for s in range(4):
        X, x, K = _stress(n, 0.1 + 0.05 * s, 0.1 * s, 50 * n + s)
        check_against_cv2(X, x, K)


# ----------------------------------------------------------------------------- fixture sets
@pytest.mark.parametrize("name", sorted(WAVE_SPECS))
def test_wave_sets(name):
    wave_set(name)


@pytest.mark.parametrize("name", DEGENERATE)
def test_degenerate_sets(name):
    degenerate_set(name)


def test_threshold_boundary_set():
    threshold_set()


# ----------------------------------------------------------------------------- the mono branch at n == 5
def mono_five_sets(count=120):
    for s in range(count):
        p0, p1, focal, pp = synth.essential_stress_set(5, 0.05 * (s % 5), 0.0, 3000 + s)
        yield p0, p1, focal, pp


def cv2_mono_or_none(p0, p1, focal, pp):
    """findEssentialMat + recoverPose; None where recoverPose raises (a stack of candidates, or no E)."""
    E, mask = cv2.findEssentialMat(p0, p1, focal, pp, cv2.RANSAC, 0.999, 1.0)
    try:
        _, R, _, _ = cv2.recoverPose(E, p0, p1, focal=focal, pp=pp, mask=mask.copy())
    except cv2.error:
        return None, None if E is None else E.shape[0] // 3
    return (R, mask.ravel().astype(bool)), 1


def test_mono_five_points_refuse_where_cv2_aborts(built):
    """n == 5: cv2 findEssentialMat returns every candidate stacked and recoverPose asserts unless there is exactly one.
    The oracle and the host build of the kernels' math refuse exactly there; on a single-candidate set (if the seed search
    finds one) the rotation and the all-ones mask agree."""
    L = _hostcheck()
    L.vo_hostcheck_mono_rotation.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_double] * 5 + [C.c_int] + [C.c_void_p] * 4
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    single = refused = 0
    for p0, p1, focal, pp in mono_five_sets():
        ref, ncand = cv2_mono_or_none(p0, p1, focal, pp)
        Ro, mo, iters = er.mono_rotation(p0, p1, focal, pp)
        E = np.zeros(9); mh = np.zeros(5, np.uint8); Rh = np.zeros(9); it = C.c_int(-1)
        good = L.vo_hostcheck_mono_rotation(p(p0), p(p1), 5, focal, pp[0], pp[1], 0.999, 1.0, 1000, p(E), p(mh), p(Rh), C.byref(it))
        assert iters == 0 and it.value == 0
        if ref is None:
            assert Ro is None and good == 0, ncand
            refused += 1
            continue
        R, mask = ref
        assert np.all(mask) and np.all(mo) and np.all(mh) and good == 5
        assert np.abs(Ro - R).max() <= 1e-6 and np.abs(Rh.reshape(3, 3) - R).max() <= 1e-6
        single += 1
    print(f"mono n == 5: {refused} sets refused, {single} single-candidate sets agree")
    assert refused > 0
