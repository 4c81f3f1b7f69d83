"""The Levenberg-Marquardt refinement at the end of solvePnPRansac (CvLevMarq inside solvePnP(ITERATIVE,
useExtrinsicGuess=true)), at its inlier-count, step-rejection and iteration-cap edges: oracle/pnp_ref.lm_refine against
cv2.solvePnP and against an independent float64 optimum (scipy.optimize.least_squares), and the kernel's step solve
(vomath::lm_solve6, host build) against OpenCV's SVD solve.

Three families of correspondence sets, built here and imported by tests/test_gpu_pnp_refine.py:
  A  driving-like sets: the stress cases of test_gpu_stages.py; 6 .. 8192 inliers around the 32-lane warps and the
     256-point chunks of k_pnp_finalize, all inliers and with outliers at a fixed stride (so that inlier indices cross the
     chunks), the latter from t_prev = 0 (the reference's first frame: |prev_param| = 0 in the first termination test);
     rotations of 0.3 .. 1.2 rad away from the small-angle Jacobian.  Some sets reject LM steps, some none.
  B  far or narrow point clusters (0.5 .. 30 m wide at 50 .. 800 m) that stop on the relative-step test.  The parameters
     are poorly determined along flat directions there, so the cost is what is compared.
  C  0.5 m clusters at 200 .. 800 m from a guess 2 m off: the refinement runs into the 20-iteration cap with at least 10
     rejected steps, and cv2's own result is not at the optimum, so cv2 is the reference.
"""
import ctypes as C
import functools

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from oracle import pnp_ref as P  # noqa: E402
from visual_odom_b200 import synth  # noqa: E402
import test_oracle_pnp_edges as E  # noqa: E402

K = synth.proj_matrices()[0][:, :3].copy()
K64 = K.astype(np.float64)
W, H = 1241, 376
T_ZERO = np.zeros(3)

STRESS = [(1500, 0.05, 0.1, 0), (1500, 0.15, 0.3, 1), (1500, 0.2, 0.5, 2), (1500, 0.25, 0.6, 3), (300, 0.1, 0.2, 4),
          (60, 0.3, 0.4, 5)]                        # test_gpu_stages.py's cases that reach the refinement (n > 5)
COUNTS = (6, 31, 32, 33, 255, 256, 257, 511, 512, 513, 2048, 8192)
STRIDE = 5                                          # every 5th correspondence an outlier
CAPACITY = 8192                                     # the GPU tests' context (max_features)
# (axis, angle rad) of the rotated sets.  About the camera's y axis (and the mixed axis) the refinement from rvec = 0 stops
# converging above ~0.6 rad and runs into the cap: those belong to no family here.
ROTATIONS = [("z", 0.3), ("z", 0.6), ("z", 0.9), ("z", 1.2), ("x", 0.9), ("x", 1.2), ("m", 0.3), ("m", 0.6)]
AXES = {"x": np.array([1.0, 0.0, 0.0]), "z": np.array([0.0, 0.0, 1.0]), "m": np.array([0.3, 1.0, -0.2]) / np.sqrt(1.13)}
FAR = [(50, 2.0), (100, 10.0), (200, 30.0), (400, 5.0), (800, 30.0), (300, 2.0), (150, 0.5)]   # (depth m, width m)
# (n, depth m, seed) of sets whose refinement runs into the cap (found by a seed search over the recipe of _cap_set)
CAP = [(44, 800, 0), (80, 400, 8), (150, 600, 6), (292, 600, 0), (292, 800, 0)]


def _scene(n, rvec, tvec, depth, width, sigma, clip, seed, outliers=None):
    """n correspondences seen by the camera at (rvec, tvec): points drawn in that camera's frame (a cluster `width` wide
    around `depth`, or the whole image at depths 6 .. 80 m when width is None) and mapped back to the world, pixel noise
    N(0, sigma) clipped to +-clip, and a gross offset of 5 .. 15 px where `outliers` is True."""
    rng = np.random.default_rng(seed)
    if width is None:
        z = rng.uniform(6, 80, n)
        uv = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1)
        Xc = np.stack([(uv[:, 0] - K64[0, 2]) / K64[0, 0] * z, (uv[:, 1] - K64[1, 2]) / K64[1, 1] * z, z], 1)
    else:
        Xc = rng.uniform(-width / 2, width / 2, (n, 3)) + np.array([0.0, 0.0, depth])
    R = P.rodrigues(rvec)
    X = ((Xc - np.asarray(tvec, np.float64)) @ R).astype(np.float32)          # R^T (Xc - t)
    x = P.project_points(X, rvec, tvec, K64) + np.clip(rng.normal(0, sigma, (n, 2)), -clip, clip)
    if outliers is not None:
        m = int(outliers.sum())
        x[outliers] += rng.uniform(5, 15, (m, 2)) * rng.choice([-1.0, 1.0], (m, 2))
    return np.ascontiguousarray(X), np.ascontiguousarray(x, np.float32)


def _strided(count):
    """Outlier mask with every STRIDE-th entry set and exactly `count` entries clear; at most CAPACITY entries (the
    8192 count becomes 6554 inliers among 8192 correspondences)."""
    total = min(count + count // (STRIDE - 1) + 1, CAPACITY)
    mask = np.arange(total) % STRIDE == STRIDE - 1
    while (~mask).sum() > count:
        total -= 1
        mask = mask[:total]
    return mask


def _specs():
    A = {}
    for n, sigma, outl, seed in STRESS:
        A[f"stress_{n}_{seed}"] = ("stress", (n, sigma, outl, seed), E.T_PREV)
    for n in COUNTS:
        A[f"all_{n}"] = ("scene", (n, synth.EGO_RVEC, synth.EGO_T, None, None, 0.01, 0.02, n, None), E.T_PREV)
        out = _strided(n)
        A[f"stride_{int((~out).sum())}"] = ("scene", (len(out), synth.EGO_RVEC, synth.EGO_T, None, None, 0.01, 0.02,
                                                     100 + n, out), T_ZERO)
    for ax, a in ROTATIONS:
        A[f"rot_{ax}_{a}"] = ("scene", (400, a * AXES[ax], synth.EGO_T, None, None, 0.1, 0.2, int(a * 10), None), E.T_PREV)
    B = {}
    for depth, width in FAR:
        t = np.array([0.1, -0.05, -1.0])
        B[f"far_{depth}_{width}"] = ("scene", (150, synth.EGO_RVEC, t, depth, width, 0.1, 0.2, depth + int(width * 10),
                                               None), t + np.array([0.05, 0.02, 0.2]))
    Cc = {}
    for n, depth, seed in CAP:
        Cc[f"cap_{n}_{depth}"] = ("cap", (n, depth, seed), None)
    return {"A": A, "B": B, "C": Cc}


def _cap_set(n, depth, seed):
    rng = np.random.default_rng(10_000 + seed)
    t = np.array([0.1, -0.05, -1.0])
    X, x = _scene(n, synth.EGO_RVEC, t, depth, 0.5, 0.1, 0.2, seed)
    d = rng.normal(size=3)
    return X, x, t + 2.0 * d / np.linalg.norm(d)


SPECS = _specs()
FAMILIES = {f: sorted(s) for f, s in SPECS.items()}
ALL = [(f, name) for f in "ABC" for name in FAMILIES[f]]


@functools.lru_cache(maxsize=None)
def lm_set(family, name):
    """(X, x, t_prev) of one set."""
    kind, args, t_prev = SPECS[family][name]
    if kind == "stress":
        X, x = E._stress(*args)[:2]
    elif kind == "scene":
        X, x = _scene(*args)
    else:
        X, x, t_prev = _cap_set(*args)
    return X, x, np.asarray(t_prev, np.float64)


@functools.lru_cache(maxsize=None)
def cv2_ransac(family, name):
    """cv2.solvePnPRansac as the reference calls it: (ok, rvec, tvec, inliers)."""
    X, x, t_prev = lm_set(family, name)
    return E.cv2_pnp(X, x, K, t_prev)


@functools.lru_cache(maxsize=None)
def oracle_ransac(family, name):
    X, x, t_prev = lm_set(family, name)
    return E.oracle_pnp(X, x, K, t_prev)


def cv2_refine(X, x, t_prev):
    """cv2.solvePnP(ITERATIVE, useExtrinsicGuess) from (rvec 0, t_prev): the refinement solvePnPRansac ends with."""
    rv = np.zeros((3, 1)); tv = np.asarray(t_prev, np.float64).reshape(3, 1).copy()
    ok, rv, tv = cv2.solvePnP(np.ascontiguousarray(X, np.float32).reshape(-1, 1, 3),
                              np.ascontiguousarray(x, np.float32).reshape(-1, 1, 2), K, np.zeros((4, 1)), rv, tv, True,
                              cv2.SOLVEPNP_ITERATIVE)
    assert ok
    return rv.ravel(), tv.ravel()


@functools.lru_cache(maxsize=None)
def refined(family, name):
    """On cv2's RANSAC inliers: dict(inl, cv2 = (rvec, tvec) of cv2.solvePnP, oracle = lm_refine's, trace)."""
    X, x, t_prev = lm_set(family, name)
    ok, _, _, inl = cv2_ransac(family, name)
    assert ok and len(inl) > 5, (family, name, len(inl))
    Xi, xi = X[inl], x[inl]
    trace = {}
    orc = P.lm_refine(Xi, xi, K64, np.zeros(3), t_prev, trace=trace)
    return dict(inl=inl, cv2=cv2_refine(Xi, xi, t_prev), oracle=orc, trace=trace)


def residuals(p, X, x):
    """Pixel residuals of the pose p = (rvec, tvec) in float64 (f32 inputs widened), cv::projectPoints' arithmetic."""
    return (P.project_points(X, p[:3], p[3:], K64) - np.asarray(x, np.float32).astype(np.float64)).ravel()


def cost(p, X, x):
    r = residuals(np.asarray(p, np.float64), X, x)
    return float(r @ r)


@functools.lru_cache(maxsize=None)
def optimum(family, name):
    """An independent float64 optimum of the refinement's objective on cv2's inliers: scipy's MINPACK Levenberg-Marquardt
    started from cv2's result -> (parameters, cost)."""
    from scipy.optimize import least_squares
    X, x, _ = lm_set(family, name)
    r = refined(family, name)
    Xi, xi = X[r["inl"]], x[r["inl"]]
    p0 = np.concatenate(r["cv2"])
    sol = least_squares(residuals, p0, args=(Xi, xi), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    return sol.x, cost(sol.x, Xi, xi)


def pdist(a, b):
    """max |a - b| over (rvec, tvec) and the scale max(1, |p|) the C family is compared at."""
    a = np.concatenate(a); b = np.concatenate(b)
    return float(np.abs(a - b).max()), max(1.0, float(np.abs(b).max()))


# ----------------------------------------------------------------------------- the families reach their edges
def test_families_reach_their_edges():
    A = [refined("A", n)["trace"] for n in FAMILIES["A"]]
    assert any(t["rejected"] > 0 for t in A) and any(t["rejected"] == 0 for t in A)
    for name in FAMILIES["B"]:
        t = refined("B", name)["trace"]
        assert t["stop"] == "eps", (name, t)
    for name in FAMILIES["C"]:
        t = refined("C", name)["trace"]
        assert t["stop"] == "cap" and t["iters"] == 20 and t["rejected"] >= 10, (name, t)
    for name in FAMILIES["A"]:
        if name.startswith(("all_", "stride_")):
            n = int(name.split("_")[1])
            assert len(cv2_ransac("A", name)[3]) == n, name        # the inlier count the set is named for


# ----------------------------------------------------------------------------- lm_refine against cv2 and the optimum
@pytest.mark.parametrize("family", "AC")
def test_lm_refine_matches_cv2(family):
    """A: 1e-9 absolute; C (at the cap, |p| up to ~1e3): 1e-8 max(1, |p|)."""
    worst = 0.0
    for name in FAMILIES[family]:
        r = refined(family, name)
        d, scale = pdist(r["oracle"], r["cv2"])
        tol = 1e-9 if family == "A" else 1e-8 * scale
        assert d <= tol, (name, d, r["trace"])
        worst = max(worst, d / (1.0 if family == "A" else scale))
    print(f"family {family}: worst lm_refine vs cv2 = {worst:.2e}")


@pytest.mark.parametrize("family", "AB")
def test_cost_is_the_float64_optimum(family):
    """The cost of cv2's result and of lm_refine's within 1e-10 relative of the optimum's."""
    worst = 0.0
    for name in FAMILIES[family]:
        X, x, _ = lm_set(family, name)
        r = refined(family, name)
        Xi, xi = X[r["inl"]], x[r["inl"]]
        c_opt = min(optimum(family, name)[1], cost(np.concatenate(r["cv2"]), Xi, xi))
        for who in ("cv2", "oracle"):
            rel = (cost(np.concatenate(r[who]), Xi, xi) - c_opt) / c_opt
            assert rel <= 1e-10, (name, who, rel)
            worst = max(worst, rel)
    print(f"family {family}: worst relative cost above the optimum = {worst:.2e}")


# ----------------------------------------------------------------------------- the kernel's step solve
def normal_equations(X, x, p):
    """J^T J and J^T e of the refinement at p (the sums k_pnp_finalize accumulates), via the oracle's Rodrigues Jacobian."""
    X = np.asarray(X, np.float32).astype(np.float64)
    R = P.rodrigues(p[:3])
    Xc = X @ R.T + p[3:]
    z = 1.0 / Xc[:, 2]
    xn, yn = Xc[:, 0] * z, Xc[:, 1] * z
    J = np.zeros((2 * len(X), 6))
    dRdr = P.rodrigues_jac(p[:3])
    for j in range(3):
        d = X @ dRdr[j].reshape(3, 3).T
        J[0::2, j] = K64[0, 0] * z * (d[:, 0] - xn * d[:, 2])
        J[1::2, j] = K64[1, 1] * z * (d[:, 1] - yn * d[:, 2])
    J[0::2, 3] = K64[0, 0] * z; J[0::2, 5] = -K64[0, 0] * xn * z
    J[1::2, 4] = K64[1, 1] * z; J[1::2, 5] = -K64[1, 1] * yn * z
    e = residuals(p, X.astype(np.float32), x)
    return J.T @ J, J.T @ e


def damped(JtJ, lam):
    A = np.array(JtJ, np.float64)
    for k in range(6):
        A[k, k] *= 1.0 + lam
    return A


def _lm_solve6():
    from visual_odom_b200 import build
    L = C.CDLL(build.build_hostcheck())
    L.vo_hostcheck_lm_solve6.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    L.vo_hostcheck_lm_solve6.restype = C.c_int

    def solve(JtJ, JtErr, lam):
        A = np.ascontiguousarray(JtJ, np.float64); b = np.ascontiguousarray(JtErr, np.float64); dx = np.zeros(6)
        chol = L.vo_hostcheck_lm_solve6(A.ctypes.data, b.ctypes.data, lam, dx.ctypes.data)
        return dx, bool(chol)
    return solve


LAMBDAS = (1e-16, 1e-3, 1.0, 1e3)


def _systems(family):
    """(name, JtJ, JtErr, lambda) at the start (rvec 0, t_prev) and at cv2's result of every set of the family."""
    for name in FAMILIES[family]:
        X, x, t_prev = lm_set(family, name)
        r = refined(family, name)
        for p in (np.concatenate([np.zeros(3), t_prev]), np.concatenate(r["cv2"])):
            JtJ, JtErr = normal_equations(X[r["inl"]], x[r["inl"]], p)
            for lam in LAMBDAS:
                yield name, JtJ, JtErr, lam


def test_step_solve_equals_svd_solve_on_driving_systems(built):
    """Family A's damped normal equations: the Cholesky step within 1e-12 relative of cv::solve(DECOMP_SVD)."""
    solve = _lm_solve6()
    worst = 0.0
    for name, JtJ, JtErr, lam in _systems("A"):
        dx, chol = solve(JtJ, JtErr, lam)
        ref = P.solve_svd(damped(JtJ, lam), JtErr)
        assert chol, name
        rel = np.abs(dx - ref).max() / np.abs(ref).max()
        assert rel <= 1e-12, (name, lam, rel)
        worst = max(worst, rel)
    print(f"family A: worst step vs SVD solve = {worst:.2e}")


def test_step_solve_backward_error_on_ill_conditioned_systems(built):
    """B's and C's systems are badly conditioned (condition numbers up to ~2e13): the Cholesky and SVD solutions differ by
    about cond * eps there, so both are held to a normwise backward error |A dx - b| / (|A| |dx| + |b|) of a few eps.
    The residual relative to |b| alone is no yardstick at these condition numbers: OpenCV's own SVD solve leaves up to
    ~3e-10 of |b| (the Cholesky solve ~2e-10)."""
    solve = _lm_solve6()
    worst = {"chol": 0.0, "svd": 0.0}
    conds = []
    for family in "BC":
        for name, JtJ, JtErr, lam in _systems(family):
            A = damped(JtJ, lam)
            dx, chol = solve(JtJ, JtErr, lam)
            for who, sol in (("chol", dx), ("svd", P.solve_svd(A, JtErr))):
                be = np.linalg.norm(A @ sol - JtErr) / (np.linalg.norm(A, 2) * np.linalg.norm(sol) + np.linalg.norm(JtErr))
                assert be <= 1e-15, (name, lam, who, be, np.linalg.cond(A))
                worst[who] = max(worst[who], be)
            conds.append(np.linalg.cond(A))
    print(f"families B, C: worst normwise backward error Cholesky {worst['chol']:.2e}, SVD {worst['svd']:.2e}, "
          f"condition numbers up to {max(conds):.1e}")


def test_step_solve_falls_back_to_svd_bit_for_bit_when_rank_deficient(built):
    """Normal equations that are not positive definite (a parameter the residuals do not depend on: a zero row and column,
    which damping leaves zero) take OpenCV's SVD solve: the step equals pnp_ref.solve_svd bit for bit."""
    solve = _lm_solve6()
    X, x, t_prev = lm_set("A", "all_256")
    r = refined("A", "all_256")
    JtJ, JtErr = normal_equations(X[r["inl"]], x[r["inl"]], np.concatenate(r["cv2"]))
    cases = []
    for zero in [(j,) for j in range(6)] + [(0, 3), (2, 5), (0, 1, 2)]:
        A = JtJ.copy(); b = JtErr.copy()
        for j in zero:
            A[j, :] = 0; A[:, j] = 0; b[j] = 0
        cases += [(zero, A, b, lam) for lam in LAMBDAS]
    for zero, A, b, lam in cases:
        dx, chol = solve(A, b, lam)
        assert not chol, (zero, lam)
        assert np.array_equal(dx, P.solve_svd(damped(A, lam), b)), (zero, lam)
