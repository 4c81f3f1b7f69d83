"""
oracle/pnp_ref.py -- TEST INFRASTRUCTURE ONLY (never imported by the product path).

Pure-Python / numpy (float64) restatement of the arithmetic behind the reference's pose solve
  cv::solvePnPRansac(points3D_t0, pointsLeft_t1, K, dist=0, rvec=0, t_prev, useExtrinsicGuess=true,
                     500, 0.5, 0.999, inliers, SOLVEPNP_ITERATIVE)        reference src/visualOdometry.cpp:176-178
  cv::Rodrigues(rvec, rotation)                                            reference src/visualOdometry.cpp:188
and of the triangulation call site
  cv::triangulatePoints + cv::convertPointsFromHomogeneous                  reference src/main.cpp:170-171

The arithmetic lives in OpenCV (un-vendored third-party dependency, pinned to 4.13.0 as
installed; modules/calib3d/src/{solvepnp,ptsetreg,epnp,calibration,triangulate}.cpp,
modules/core/src/{lapack,matmul,rand}.cpp -- not on disk).  The published algorithms are restated
here and pinned against cv2 4.13.0 by tests/test_oracle_pnp.py, most of them BIT-FOR-BIT:
  * cv::SVD::compute for small matrices = one-sided Jacobi (OpenCV's own JacobiSVDImpl_, the LAPACK
    HAL is bypassed below 25 rows), scalar sequential dot products, OpenCV's scaled hypot
  * cv::solve / cv::invert with DECOMP_SVD (SVBkSb), cv::mulTransposed (sequential sums)
  * EPnP exactly as OpenCV structures it (control points by PCA, left singular vectors of the 12x12
    M^T M -- for a 5-point sample two of them span a degenerate null space, so every rounding
    matters --, beta approximations 1/2/3, 5 Gauss-Newton steps with its Householder QR, Horn alignment)
  * RNG (multiply-with-carry, state 2^64-1), 5-distinct-index subsets, adaptive niters rule
  * reprojection in f64 -> f32, squared error in f32, inlier iff err <= (float)(0.5^2)
  * final pose: Levenberg-Marquardt (CvLevMarq) on (rvec, t) over the inliers from (rvec=0, t_prev)
Pure-Python loops: only meant for the small cases the tests use.
"""
import math

import numpy as np

DBL_MIN = 2.2250738585072014e-308
DBL_EPS = 2.220446049250313e-16
FLT_EPS = 1.1920928955078125e-07

# EPnP's scalars are Python floats, whose division by zero raises where C++ yields inf / nan.  A degenerate sample (five
# identical points) is re-run with numpy float64 scalars: the same IEEE double operations, but non-finite results
# propagate as they do in OpenCV.
_fl = float

# ----------------------------------------------------------------------------- RNG
RNG_COEFF = 4164903690
MASK32 = 0xFFFFFFFF
MASK64 = 0xFFFFFFFFFFFFFFFF


class CvRNG:
    """cv::RNG: s = (uint32)s * 4164903690 + (s >> 32); next() returns (uint32)s."""

    def __init__(self, state=MASK64):
        self.state = state if state else MASK64

    def next(self):
        self.state = ((self.state & MASK32) * RNG_COEFF + (self.state >> 32)) & MASK64
        return self.state & MASK32

    def uniform(self, a, b):
        return a if a == b else int(self.next() % (b - a)) + a


def rng_raw_stream(n, state=MASK64):
    r = CvRNG(state)
    return np.array([r.next() for _ in range(n)], dtype=np.uint32)


def ransac_subset(rng, count, model_points=5):
    """RANSACPointSetRegistrator::getSubset: model_points distinct indices, redraw on duplicate."""
    idx = []
    for _ in range(model_points):
        while True:
            v = rng.uniform(0, count)
            if v not in idx:
                break
        idx.append(v)
    return idx


def ransac_update_num_iters(p, ep, model_points, max_iters):
    """cv::RANSACUpdateNumIters"""
    p = min(max(p, 0.0), 1.0)
    ep = min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, DBL_MIN)
    denom = 1.0 - (1.0 - ep) ** model_points      # std::pow(1 - ep, modelPoints)
    if denom < DBL_MIN:
        return 0
    num = math.log(num)
    denom = math.log(denom)
    if denom >= 0 or -num >= max_iters * (-denom):
        return max_iters
    return int(np.rint(num / denom))      # cvRound: round-half-even


# ----------------------------------------------------------------------------- small dense linear algebra
def _hypot(a, b):
    """OpenCV's own hypot (lapack.cpp), not libm's."""
    a = abs(a); b = abs(b)
    if a > b:
        b /= a
        return a * math.sqrt(1 + b * b)
    if b > 0:
        a /= b
        return b * math.sqrt(1 + a * a)
    return 0.0


def jacobi_svd_t(At, m, n, n1):
    """JacobiSVDImpl_<double>(At, W, Vt, m, n, n1, DBL_MIN, DBL_EPSILON*10).
    At: n rows of length m (= A^T).  Returns (W[n], At_out = U^T rows, Vt)."""
    eps = DBL_EPS * 10
    At = [[_fl(v) for v in r] for r in At]
    W = [0.0] * n
    Vt = [[1.0 if i == k else 0.0 for k in range(n)] for i in range(n)]
    for i in range(n):
        sd = 0.0
        for k in range(m):
            t = At[i][k]
            sd += t * t
        W[i] = sd
    for _ in range(max(m, 30)):
        changed = False
        for i in range(n - 1):
            for j in range(i + 1, n):
                Ai, Aj = At[i], At[j]
                a, b, p = W[i], W[j], 0.0
                for k in range(m):
                    p += Ai[k] * Aj[k]
                if abs(p) <= eps * math.sqrt(a * b):
                    continue
                p *= 2
                beta = a - b
                gamma = _hypot(p, beta)
                if beta < 0:
                    delta = (gamma - beta) * 0.5
                    s = math.sqrt(delta / gamma)
                    c = p / (gamma * s * 2)
                else:
                    c = math.sqrt((gamma + beta) / (gamma * 2))
                    s = p / (gamma * c * 2)
                a = b = 0.0
                for k in range(m):
                    t0 = c * Ai[k] + s * Aj[k]
                    t1 = -s * Ai[k] + c * Aj[k]
                    Ai[k] = t0; Aj[k] = t1
                    a += t0 * t0; b += t1 * t1
                W[i] = a; W[j] = b
                changed = True
                Vi, Vj = Vt[i], Vt[j]
                for k in range(n):
                    t0 = c * Vi[k] + s * Vj[k]
                    t1 = -s * Vi[k] + c * Vj[k]
                    Vi[k] = t0; Vj[k] = t1
        if not changed:
            break
    for i in range(n):
        sd = 0.0
        for k in range(m):
            t = At[i][k]
            sd += t * t
        W[i] = math.sqrt(sd)
    for i in range(n - 1):
        j = i
        for k in range(i + 1, n):
            if W[j] < W[k]:
                j = k
        if i != j:
            W[i], W[j] = W[j], W[i]
            At[i], At[j] = At[j], At[i]
            Vt[i], Vt[j] = Vt[j], Vt[i]
    rng = CvRNG(0x12345678)
    for i in range(n1):
        sd = W[i] if i < n else 0.0
        ii = 0
        while ii < 100 and sd <= DBL_MIN:
            # zero singular value: random +-1/m vector, Gram-Schmidt against the previous rows
            val0 = 1.0 / m
            for k in range(m):
                At[i][k] = val0 if (rng.next() & 256) != 0 else -val0
            for _ in range(2):
                for j in range(i):
                    sd = 0.0
                    for k in range(m):
                        sd += At[i][k] * At[j][k]
                    asum = 0.0
                    for k in range(m):
                        t = At[i][k] - sd * At[j][k]
                        At[i][k] = t
                        asum += abs(t)
                    asum = 1 / asum if asum > eps * 100 else 0.0
                    for k in range(m):
                        At[i][k] *= asum
            sd = 0.0
            for k in range(m):
                t = At[i][k]
                sd += t * t
            sd = math.sqrt(sd)
            ii += 1
        s = 1 / sd if sd > DBL_MIN else 0.0
        for k in range(m):
            At[i][k] *= s
    return W, At, Vt


def svd(A):
    """cv::SVD::compute(A, w, u, vt) for m >= n (float64): returns (w[n], u m x n, vt n x n)."""
    A = np.asarray(A, np.float64)
    m, n = A.shape
    assert m >= n
    W, Ut, Vt = jacobi_svd_t(A.T.tolist(), m, n, n)
    return np.array(W), np.array(Ut).T.copy(), np.array(Vt)


def _svbksb(m, n, w, u_rows, vt_rows, b):
    """SVBkSbImpl_ with u given as U^T rows (uT=true), v as V^T rows (vT=true), nb == 1 or b None."""
    nm = min(m, n)
    threshold = 0.0
    for i in range(nm):
        threshold += w[i]
    threshold *= DBL_EPS * 2
    if b is not None:
        x = [0.0] * n
        for i in range(nm):
            wi = w[i]
            if abs(wi) <= threshold:
                continue
            wi = 1 / wi
            s = 0.0
            for j in range(m):
                s += u_rows[i][j] * b[j]
            s *= wi
            for j in range(n):
                x[j] = x[j] + s * vt_rows[i][j]
        return x
    # b == NULL: x = V diag(1/w) U^T   (n x m)
    x = [[0.0] * m for _ in range(n)]
    for i in range(nm):
        wi = w[i]
        if abs(wi) <= threshold:
            continue
        wi = 1 / wi
        buf = [u_rows[i][j] * wi for j in range(m)]
        for r in range(n):
            s = vt_rows[i][r]
            for j in range(m):
                x[r][j] = x[r][j] + s * buf[j]
    return x


def solve_svd(A, b):
    """cv::solve(A, b, x, DECOMP_SVD), single right-hand side."""
    A = np.asarray(A, np.float64)
    m, n = A.shape
    W, Ut, Vt = jacobi_svd_t(A.T.tolist(), m, n, n)
    return np.array(_svbksb(m, n, W, Ut, Vt, [_fl(v) for v in b]))


def invert_svd(A):
    """cv::invert(A, Ainv, DECOMP_SVD) for square A."""
    A = np.asarray(A, np.float64)
    n = A.shape[0]
    W, Ut, Vt = jacobi_svd_t(A.T.tolist(), n, n, n)
    return np.array(_svbksb(n, n, W, Ut, Vt, None))


def mul_transposed(M):
    """cv::mulTransposed(M, dst, aTa=true) (small-matrix path): M^T M, sequential sums over rows."""
    M = np.asarray(M, np.float64)
    rows, cols = M.shape
    out = np.zeros((cols, cols))
    for i in range(cols):
        for j in range(i, cols):
            s = 0.0
            for k in range(rows):
                s += M[k, i] * M[k, j]
            out[i, j] = s
            out[j, i] = s
    return out


# ----------------------------------------------------------------------------- Rodrigues / projection
def rodrigues(rvec):
    """cv::Rodrigues vector -> matrix (f64)."""
    rx, ry, rz = (float(v) for v in np.asarray(rvec, np.float64).reshape(3))
    theta = math.sqrt(rx * rx + ry * ry + rz * rz)
    if theta < DBL_EPS:
        return np.eye(3)
    c = math.cos(theta); s = math.sin(theta); c1 = 1.0 - c
    itheta = 1.0 / theta if theta else 0.0
    rx *= itheta; ry *= itheta; rz *= itheta
    rrt = [rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz]
    r_x = [0.0, -rz, ry, rz, 0.0, -rx, -ry, rx, 0.0]
    eye = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    return np.array([c * eye[k] + c1 * rrt[k] + s * r_x[k] for k in range(9)]).reshape(3, 3)


def rodrigues_jac(rvec):
    """dR/dr as OpenCV lays it out (3 x 9: d vec(R) / d r_i in row i)."""
    r = np.asarray(rvec, np.float64).reshape(3)
    theta = math.sqrt(float(r @ r))
    J = np.zeros((3, 9))
    if theta < DBL_EPS:
        J[0, 5] = -1; J[0, 7] = 1
        J[1, 2] = 1; J[1, 6] = -1
        J[2, 1] = -1; J[2, 3] = 1
        return J
    c = math.cos(theta); s = math.sin(theta); c1 = 1.0 - c
    itheta = 1.0 / theta
    k = r * itheta
    rrt = np.outer(k, k)
    r_x = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    I = np.eye(3)
    drrt = np.array([[2 * k[0], k[1], k[2], k[1], 0, 0, k[2], 0, 0],
                     [0, k[0], 0, k[0], 2 * k[1], k[2], 0, k[2], 0],
                     [0, 0, k[0], 0, 0, k[1], k[0], k[1], 2 * k[2]]], np.float64)
    d_r_x = np.array([[0, 0, 0, 0, 0, -1, 0, 1, 0],
                      [0, 0, 1, 0, 0, 0, -1, 0, 0],
                      [0, -1, 0, 1, 0, 0, 0, 0, 0]], np.float64)
    for i in range(3):
        ri = k[i]
        a0 = -s * ri; a1 = (s - 2 * c1 * itheta) * ri; a2 = c1 * itheta
        a3 = (c - s * itheta) * ri; a4 = s * itheta
        J[i] = (a0 * I + a1 * rrt + a3 * r_x).ravel() + a2 * drrt[i] + a4 * d_r_x[i]
    return J


def rodrigues_inv(R):
    """cv::Rodrigues matrix -> vector (f64).  An entry outside [-100, 100) or non-finite gives the zero vector
    (OpenCV's checkRange guard)."""
    R = np.asarray(R, np.float64)
    if not np.all((R >= -100) & (R < 100)):
        return np.zeros(3)
    _, U, Vt = svd(R)
    Rm = np.zeros((3, 3))
    for i in range(3):
        for j in range(3):
            s = 0.0
            for k in range(3):
                s += U[i, k] * Vt[k, j]
            Rm[i, j] = s
    R = Rm
    rx = R[2, 1] - R[1, 2]; ry = R[0, 2] - R[2, 0]; rz = R[1, 0] - R[0, 1]
    s = math.sqrt((rx * rx + ry * ry + rz * rz) * 0.25)
    c = (R[0, 0] + R[1, 1] + R[2, 2] - 1) * 0.5
    c = 1.0 if c > 1.0 else (-1.0 if c < -1.0 else c)
    theta = math.acos(c)
    if s < 1e-5:
        if c > 0:
            return np.zeros(3)
        t = (R[0, 0] + 1) * 0.5
        rx = math.sqrt(max(t, 0.0))
        t = (R[1, 1] + 1) * 0.5
        ry = math.sqrt(max(t, 0.0)) * (-1.0 if R[0, 1] < 0 else 1.0)
        t = (R[2, 2] + 1) * 0.5
        rz = math.sqrt(max(t, 0.0)) * (-1.0 if R[0, 2] < 0 else 1.0)
        if abs(rx) < abs(ry) and abs(rx) < abs(rz) and (R[1, 2] > 0) != (ry * rz > 0):
            rz = -rz
        theta /= math.sqrt(rx * rx + ry * ry + rz * rz)
        return np.array([rx * theta, ry * theta, rz * theta])
    vth = 1 / (2 * s)
    vth *= theta
    return np.array([rx * vth, ry * vth, rz * vth])


def project_points(X, rvec, tvec, K):
    """cv::projectPoints with zero distortion, f64 arithmetic in OpenCV's operation order; (N,2) f64."""
    R = rodrigues(rvec)
    X = np.asarray(X, np.float64).reshape(-1, 3)
    t = np.asarray(tvec, np.float64).reshape(3)
    x = R[0, 0] * X[:, 0] + R[0, 1] * X[:, 1] + R[0, 2] * X[:, 2] + t[0]
    y = R[1, 0] * X[:, 0] + R[1, 1] * X[:, 1] + R[1, 2] * X[:, 2] + t[1]
    z = R[2, 0] * X[:, 0] + R[2, 1] * X[:, 1] + R[2, 2] * X[:, 2] + t[2]
    with np.errstate(divide="ignore"):
        z = np.where(z != 0, 1.0 / z, 1.0)
    x = x * z
    y = y * z
    return np.stack([x * K[0, 0] + K[0, 2], y * K[1, 1] + K[1, 2]], axis=1)


def reproj_err_f32(X, x, rvec, tvec, K):
    """PnPRansacCallback::computeError: projections stored f32, squared distance in f32."""
    p = project_points(X, rvec, tvec, K).astype(np.float32)
    d = np.asarray(x, np.float32).reshape(-1, 2) - p
    dx2 = d[:, 0] * d[:, 0]
    dy2 = d[:, 1] * d[:, 1]
    return (dx2 + dy2).astype(np.float32)


# ----------------------------------------------------------------------------- triangulation
def triangulate(P_l, P_r, pts_l, pts_r):
    """cv::triangulatePoints (per-point 4x4 DLT, last row of V^T, stored f32) followed by
    cv::convertPointsFromHomogeneous (f32: scale = 1/w where |w| > FLT_EPSILON, else 1; x*scale)."""
    Pl = np.asarray(P_l, np.float32).astype(np.float64)
    Pr = np.asarray(P_r, np.float32).astype(np.float64)
    a = np.asarray(pts_l, np.float32).reshape(-1, 2)
    b = np.asarray(pts_r, np.float32).reshape(-1, 2)
    n = len(a)
    X4 = np.zeros((n, 4), np.float32)
    for i in range(n):
        x, y, xr, yr = float(a[i, 0]), float(a[i, 1]), float(b[i, 0]), float(b[i, 1])
        A = np.array([x * Pl[2] - Pl[0], y * Pl[2] - Pl[1], xr * Pr[2] - Pr[0], yr * Pr[2] - Pr[1]])
        _, _, vt = svd(A)
        X4[i] = vt[3].astype(np.float32)
    return dehomogenize_f32(X4)


def dehomogenize_f32(X4):
    """cv::convertPointsFromHomogeneous on f32 4-vectors: it divides only where |w| > FLT_EPSILON (strictly, so
    |w| == FLT_EPSILON and a NaN w keep scale 1).  A zero-disparity point (w ~ 1e-18) stays the unit-norm column."""
    X4 = np.asarray(X4, np.float32)
    w = X4[:, 3]
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        scale = np.where(np.abs(w) > np.finfo(np.float32).eps, np.float32(1.0) / w, np.float32(1.0)).astype(np.float32)
    return (X4[:, :3] * scale[:, None]).astype(np.float32)


# ----------------------------------------------------------------------------- EPnP
def undistort_normalize_f32(x, K):
    """cv::undistortPoints with zero distortion: ((u - cx) * (1/fx)) in f64, stored f32."""
    x = np.asarray(x, np.float32).reshape(-1, 2).astype(np.float64)
    ifx = 1.0 / K[0, 0]
    ify = 1.0 / K[1, 1]
    return np.stack([(x[:, 0] - K[0, 2]) * ifx, (x[:, 1] - K[1, 2]) * ify], 1).astype(np.float32)


def _dot3(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _qr_solve_6x4(A, b):
    """epnp::qr_solve (Householder, including its off-by-one column-scale scan)."""
    nr, nc = 6, 4
    A = [_fl(v) for v in np.asarray(A, np.float64).ravel()]
    b = [_fl(v) for v in b]
    A1 = [0.0] * nr
    A2 = [0.0] * nr
    for k in range(nc):
        kk = k * nc + k
        eta = abs(A[kk])
        p = kk
        for i in range(k + 1, nr):
            elt = abs(A[p])
            if eta < elt:
                eta = elt
            p += nc
        if eta == 0:
            return None
        inv_eta = 1.0 / eta
        sum2 = 0.0
        p = kk
        for i in range(k, nr):
            A[p] *= inv_eta
            sum2 += A[p] * A[p]
            p += nc
        sigma = math.sqrt(sum2)
        if A[kk] < 0:
            sigma = -sigma
        A[kk] += sigma
        A1[k] = sigma * A[kk]
        A2[k] = -eta * sigma
        for j in range(k + 1, nc):
            p = kk
            s = 0.0
            for i in range(k, nr):
                s += A[p] * A[p + j - k]
                p += nc
            tau = s / A1[k]
            p = kk
            for i in range(k, nr):
                A[p + j - k] -= tau * A[p]
                p += nc
    for j in range(nc):
        jj = j * nc + j
        p = jj
        tau = 0.0
        for i in range(j, nr):
            tau += A[p] * b[i]
            p += nc
        tau /= A1[j]
        p = jj
        for i in range(j, nr):
            b[i] -= tau * A[p]
            p += nc
    X = [0.0] * nc
    X[nc - 1] = b[nc - 1] / A2[nc - 1]
    for i in range(nc - 2, -1, -1):
        s = 0.0
        for j in range(i + 1, nc):
            s += A[i * nc + j] * X[j]
        X[i] = (b[i] - s) / A2[i]
    return X


def epnp(X, x, K):
    """cv::solvePnP(..., SOLVEPNP_EPNP) with zero distortion: returns (rvec, tvec) float64."""
    global _fl
    try:
        return _epnp(X, x, K)
    except ZeroDivisionError:
        _fl = np.float64
        try:
            with np.errstate(all="ignore"):
                rv, tv = _epnp(X, x, K)
            return np.asarray(rv, np.float64), np.asarray(tv, np.float64)
        finally:
            _fl = float


def _epnp(X, x, K):
    X = np.asarray(X, np.float32).reshape(-1, 3).astype(np.float64)
    K = np.asarray(K, np.float64)
    n = len(X)
    fu, fv, uc, vc = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    xn = undistort_normalize_f32(x, K).astype(np.float64)
    us = np.stack([xn[:, 0] * fu + uc, xn[:, 1] * fv + vc], 1)
    X = [[_fl(v) for v in row] for row in X]
    us = [[_fl(v) for v in row] for row in us]
    # choose_control_points
    cws = [[0.0] * 3 for _ in range(4)]
    for i in range(n):
        for j in range(3):
            cws[0][j] += X[i][j]
    for j in range(3):
        cws[0][j] /= n
    pw0 = [[X[i][j] - cws[0][j] for j in range(3)] for i in range(n)]
    dc, uc_mat, _ = svd(mul_transposed(pw0))
    uct = uc_mat.T
    for i in range(1, 4):
        k = math.sqrt(dc[i - 1] / n)
        for j in range(3):
            cws[i][j] = cws[0][j] + k * uct[i - 1][j]
    # compute_barycentric_coordinates
    cc = [[cws[j + 1][i] - cws[0][i] for j in range(3)] for i in range(3)]
    ci = invert_svd(cc)
    al = [[0.0] * 4 for _ in range(n)]
    for i in range(n):
        for j in range(3):
            al[i][1 + j] = ci[j][0] * (X[i][0] - cws[0][0]) + ci[j][1] * (X[i][1] - cws[0][1]) + \
                           ci[j][2] * (X[i][2] - cws[0][2])
        al[i][0] = 1.0 - al[i][1] - al[i][2] - al[i][3]
    # M and its Gram matrix
    M = np.zeros((2 * n, 12))
    for i in range(n):
        for j in range(4):
            M[2 * i, 3 * j] = al[i][j] * fu
            M[2 * i, 3 * j + 2] = al[i][j] * (uc - us[i][0])
            M[2 * i + 1, 3 * j + 1] = al[i][j] * fv
            M[2 * i + 1, 3 * j + 2] = al[i][j] * (vc - us[i][1])
    _, U, _ = svd(mul_transposed(M))
    ut = U.T
    v = [[_fl(t) for t in ut[11 - i]] for i in range(4)]
    pairs = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    dv = [[[v[i][3 * a + c] - v[i][3 * b + c] for c in range(3)] for (a, b) in pairs] for i in range(4)]
    L = []
    for i in range(6):
        d0, d1, d2, d3 = dv[0][i], dv[1][i], dv[2][i], dv[3][i]
        L.append([_dot3(d0, d0), 2.0 * _dot3(d0, d1), _dot3(d1, d1), 2.0 * _dot3(d0, d2), 2.0 * _dot3(d1, d2),
                  _dot3(d2, d2), 2.0 * _dot3(d0, d3), 2.0 * _dot3(d1, d3), 2.0 * _dot3(d2, d3), _dot3(d3, d3)])

    def dist2(p, q):
        return (p[0] - q[0]) * (p[0] - q[0]) + (p[1] - q[1]) * (p[1] - q[1]) + (p[2] - q[2]) * (p[2] - q[2])

    rho = [dist2(cws[a], cws[b]) for a, b in pairs]

    def cols(idx):
        return [[L[i][c] for c in idx] for i in range(6)]

    def approx1():
        b4 = solve_svd(cols([0, 1, 3, 6]), rho)
        if b4[0] < 0:
            b0 = math.sqrt(-b4[0]); return [b0, -b4[1] / b0, -b4[2] / b0, -b4[3] / b0]
        b0 = math.sqrt(b4[0]); return [b0, b4[1] / b0, b4[2] / b0, b4[3] / b0]

    def approx2():
        b3 = solve_svd(cols([0, 1, 2]), rho)
        if b3[0] < 0:
            b0 = math.sqrt(-b3[0]); b1 = math.sqrt(-b3[2]) if b3[2] < 0 else 0.0
        else:
            b0 = math.sqrt(b3[0]); b1 = math.sqrt(b3[2]) if b3[2] > 0 else 0.0
        if b3[1] < 0:
            b0 = -b0
        return [b0, b1, 0.0, 0.0]

    def approx3():
        b5 = solve_svd(cols([0, 1, 2, 3, 4]), rho)
        if b5[0] < 0:
            b0 = math.sqrt(-b5[0]); b1 = math.sqrt(-b5[2]) if b5[2] < 0 else 0.0
        else:
            b0 = math.sqrt(b5[0]); b1 = math.sqrt(b5[2]) if b5[2] > 0 else 0.0
        if b5[1] < 0:
            b0 = -b0
        return [b0, b1, b5[3] / b0, 0.0]

    def gauss_newton(be):
        be = list(be)
        for _ in range(5):
            A = [[0.0] * 4 for _ in range(6)]
            b = [0.0] * 6
            for i in range(6):
                r = L[i]
                A[i][0] = 2 * r[0] * be[0] + r[1] * be[1] + r[3] * be[2] + r[6] * be[3]
                A[i][1] = r[1] * be[0] + 2 * r[2] * be[1] + r[4] * be[2] + r[7] * be[3]
                A[i][2] = r[3] * be[0] + r[4] * be[1] + 2 * r[5] * be[2] + r[8] * be[3]
                A[i][3] = r[6] * be[0] + r[7] * be[1] + r[8] * be[2] + 2 * r[9] * be[3]
                b[i] = rho[i] - (r[0] * be[0] * be[0] + r[1] * be[0] * be[1] + r[2] * be[1] * be[1] +
                                 r[3] * be[0] * be[2] + r[4] * be[1] * be[2] + r[5] * be[2] * be[2] +
                                 r[6] * be[0] * be[3] + r[7] * be[1] * be[3] + r[8] * be[2] * be[3] +
                                 r[9] * be[3] * be[3])
            xx = _qr_solve_6x4(A, b)
            if xx is None:
                # qr_solve returns without touching x (zero-initialised once): x keeps its last value
                xx = getattr(gauss_newton, "_last", [0.0] * 4)
            gauss_newton._last = xx
            be = [be[i] + xx[i] for i in range(4)]
        return be

    def compute_R_and_t(be):
        ccs = [[0.0] * 3 for _ in range(4)]
        for i in range(4):
            for j in range(4):
                for k in range(3):
                    ccs[j][k] += be[i] * v[i][3 * j + k]
        pcs = [[al[i][0] * ccs[0][j] + al[i][1] * ccs[1][j] + al[i][2] * ccs[2][j] + al[i][3] * ccs[3][j]
                for j in range(3)] for i in range(n)]
        if pcs[0][2] < 0.0:
            ccs = [[-t for t in r] for r in ccs]
            pcs = [[-t for t in r] for r in pcs]
        pc0 = [0.0] * 3; pw0_ = [0.0] * 3
        for i in range(n):
            for j in range(3):
                pc0[j] += pcs[i][j]; pw0_[j] += X[i][j]
        for j in range(3):
            pc0[j] /= n; pw0_[j] /= n
        abt = [[0.0] * 3 for _ in range(3)]
        for i in range(n):
            for j in range(3):
                abt[j][0] += (pcs[i][j] - pc0[j]) * (X[i][0] - pw0_[0])
                abt[j][1] += (pcs[i][j] - pc0[j]) * (X[i][1] - pw0_[1])
                abt[j][2] += (pcs[i][j] - pc0[j]) * (X[i][2] - pw0_[2])
        _, u_, vt_ = svd(abt)
        v_ = vt_.T
        R = [[_dot3(u_[i], v_[j]) for j in range(3)] for i in range(3)]
        det = R[0][0] * R[1][1] * R[2][2] + R[0][1] * R[1][2] * R[2][0] + R[0][2] * R[1][0] * R[2][1] - \
            R[0][2] * R[1][1] * R[2][0] - R[0][1] * R[1][0] * R[2][2] - R[0][0] * R[1][2] * R[2][1]
        if det < 0:
            R[2] = [-t for t in R[2]]
        t = [pc0[0] - _dot3(R[0], pw0_), pc0[1] - _dot3(R[1], pw0_), pc0[2] - _dot3(R[2], pw0_)]
        s2 = 0.0
        for i in range(n):
            Xc = _dot3(R[0], X[i]) + t[0]
            Yc = _dot3(R[1], X[i]) + t[1]
            iz = 1.0 / (_dot3(R[2], X[i]) + t[2])
            ue = uc + fu * Xc * iz
            ve = vc + fv * Yc * iz
            s2 += math.sqrt((us[i][0] - ue) * (us[i][0] - ue) + (us[i][1] - ve) * (us[i][1] - ve))
        return s2 / n, np.array(R), np.array(t)

    gauss_newton._last = [0.0] * 4
    sols = [compute_R_and_t(gauss_newton(f())) for f in (approx1, approx2, approx3)]
    N = 0
    if sols[1][0] < sols[0][0]:
        N = 1
    if sols[2][0] < sols[N][0]:
        N = 2
    return rodrigues_inv(sols[N][1]), sols[N][2]


# ----------------------------------------------------------------------------- LM refinement
def lm_refine(X, x, K, rvec0, tvec0, max_iter=20, eps=FLT_EPS, trace=None):
    """cvFindExtrinsicCameraParams2's refinement: CvLevMarq over (rvec, tvec), pixel residuals.
    trace: a dict that receives iters (iterations run), rejected (steps rejected for raising the error, over all
    iterations) and stop ("cap" when max_iter ended it, "eps" when the relative step fell below eps); it changes nothing
    else."""
    X = np.asarray(X, np.float32).reshape(-1, 3).astype(np.float64)
    m = np.asarray(x, np.float32).reshape(-1, 2).astype(np.float64)
    K = np.asarray(K, np.float64)
    fx, fy = K[0, 0], K[1, 1]
    n = len(X)
    param = np.concatenate([np.asarray(rvec0, np.float64).reshape(3), np.asarray(tvec0, np.float64).reshape(3)])

    def proj(p, jac):
        r, t = p[:3], p[3:]
        R = rodrigues(r)
        Xc = X @ R.T + t
        z = np.where(Xc[:, 2] != 0, 1.0 / Xc[:, 2], 1.0)
        xn = Xc[:, 0] * z
        yn = Xc[:, 1] * z
        err = np.empty(2 * n)
        err[0::2] = xn * fx + K[0, 2] - m[:, 0]
        err[1::2] = yn * fy + K[1, 2] - m[:, 1]
        if not jac:
            return err, None
        J = np.zeros((2 * n, 6))
        dRdr = rodrigues_jac(r)                     # 3 x 9
        for j in range(3):
            dR = dRdr[j].reshape(3, 3)
            d = X @ dR.T                             # d Xc / d r_j
            J[0::2, j] = fx * z * (d[:, 0] - xn * d[:, 2])
            J[1::2, j] = fy * z * (d[:, 1] - yn * d[:, 2])
        J[0::2, 3] = fx * z; J[0::2, 5] = -fx * xn * z
        J[1::2, 4] = fy * z; J[1::2, 5] = -fy * yn * z
        return err, J

    lam_lg10 = -3
    iters = rejected = 0
    err, J = proj(param, True)
    prev_err_norm = None
    while True:
        JtJ = J.T @ J
        JtErr = J.T @ err
        prev_param = param.copy()
        if iters == 0:
            prev_err_norm = math.sqrt(float(err @ err))

        def step():
            lam = math.exp(lam_lg10 * math.log(10.0))
            A = JtJ.copy()
            A[np.diag_indices(6)] *= 1.0 + lam
            return prev_param - np.linalg.lstsq(A, JtErr, rcond=None)[0]

        param = step()
        while True:
            err, _ = proj(param, False)
            err_norm = math.sqrt(float(err @ err))
            if err_norm > prev_err_norm:
                lam_lg10 += 1
                rejected += 1
                if lam_lg10 <= 16:
                    param = step()
                    continue
            break
        lam_lg10 = max(lam_lg10 - 1, -16)
        iters += 1
        rel = np.linalg.norm(param - prev_param) / max(np.linalg.norm(prev_param), DBL_EPS)
        if iters >= max_iter or rel < eps:
            if trace is not None:
                trace.update(iters=iters, rejected=rejected, stop="eps" if rel < eps else "cap")
            break
        prev_err_norm = err_norm
        err, J = proj(param, True)
    return param[:3].copy(), param[3:].copy()


# ----------------------------------------------------------------------------- n == 4: the P3P case
def p3p_solutions(X, y):
    """All poses (R, t) with positive depths of three world points X (3 x 3) seen at normalised coordinates y (3 x 2).
    Grunert's formulation (s2 = u s1, s3 = v s1, quartic in v built from polynomial products); the solution SET is what
    cv::solveP3P returns (checked in tests/test_oracle_pnp.py), not its operation order."""
    X = np.asarray(X, np.float64)
    f = np.concatenate([np.asarray(y, np.float64), np.ones((3, 1))], 1)
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    a2 = np.sum((X[1] - X[2]) ** 2); b2 = np.sum((X[0] - X[2]) ** 2); c2 = np.sum((X[0] - X[1]) ** 2)
    if not b2 > 0:
        return []
    ca, cb, cg = f[1] @ f[2], f[0] @ f[2], f[0] @ f[1]
    Kq = (a2 - c2) / b2
    N = np.array([Kq + 1, -2 * Kq * cb, Kq - 1])          # ascending powers of v
    D = np.array([2 * cg, -2 * ca])
    Q = np.array([1, -2 * cb, 1])
    pm = np.polynomial.polynomial.polymul
    D2 = pm(D, D)
    poly = np.zeros(5)
    for term in (D2, pm(N, N), -2 * cg * pm(N, D), -(c2 / b2) * pm(Q, D2)):
        poly[:len(term)] += term
    if not np.all(np.isfinite(poly)):
        return []

    def frame(A):
        e1 = A[1] - A[0]; e1 = e1 / np.linalg.norm(e1)
        e3 = np.cross(e1, A[2] - A[0]); e3 = e3 / np.linalg.norm(e3)
        return np.stack([e1, np.cross(e3, e1), e3], 1)

    pr = poly[::-1]
    d1, d2 = np.polyder(pr), np.polyder(pr, 2)
    scale_at = lambda v: np.polyval(np.abs(pr), abs(v))

    def polish(v):
        for _ in range(4):
            dv = np.polyval(d1, v)
            if dv == 0:
                break
            v = v - np.polyval(pr, v) / dv
        return v

    # real roots of the quartic.  Two real roots that nearly coincide (poses next to Grunert's singularity, clustered points)
    # come out of a root finder with errors ~ sqrt(eps), often as a conjugate pair with a small imaginary part: such a pair is
    # re-derived from the local parabola around the extremum of the quartic (p(v) ~ A ((v - vm)^2 + s), real iff s <= 0).
    vs = []
    for r in np.roots(np.trim_zeros(pr, "f")):
        v, mag = r.real, max(1.0, abs(r.real))
        if abs(r.imag) <= 1e-9 * mag:
            vs.append(polish(v))
        elif 0 < r.imag <= 1e-3 * mag:
            vm = v
            for _ in range(4):                               # extremum: Newton on p'
                dd = np.polyval(d2, vm)
                if dd == 0:
                    break
                vm = vm - np.polyval(d1, vm) / dd
            A = 0.5 * np.polyval(d2, vm)
            if A != 0:
                sq = np.polyval(pr, vm) / A
                if sq <= 0:
                    dl = np.sqrt(-sq)
                    vs += [polish(vm - dl), polish(vm + dl)] if dl > 1e-12 * mag else [vm]
    sols, seen = [], []
    for v in vs:
        if not abs(np.polyval(pr, v)) <= 1e-9 * scale_at(v) or not v > 0:
            continue
        q = 1 + v * v - 2 * v * cb
        if not q > 0:
            continue
        # u = N(v) / D(v); next to the singularity D(v) -> 0 (N(v) -> 0 too) the quotient only selects which root of the
        # quadratic u^2 - 2 cos(gamma) u + 1 - (c^2 / b^2) q = 0 (third distance equation) belongs to this v
        Dv = D[0] + D[1] * v
        rel = abs(Dv) / (abs(D[0]) + abs(D[1] * v))
        u_lin = (N[0] + N[1] * v + N[2] * v * v) / Dv if Dv != 0 else None
        if rel > 1e-3:
            us = [u_lin]
        else:
            disc = cg * cg - 1 + (c2 / b2) * q
            uq = [cg + np.sqrt(disc), cg - np.sqrt(disc)] if disc >= 0 else []
            if uq and u_lin is not None and rel > 1e-9:
                us = [min(uq, key=lambda z: abs(z - u_lin))]
            else:
                us = uq
        for u in us:
            if not u > 0:
                continue
            if abs(u * u + v * v - 2 * u * v * ca - (a2 / b2) * q) > 1e-5 * (u * u + v * v + (a2 / b2) * q):
                continue
            if any(abs(u - a) <= 1e-7 * u and abs(v - b) <= 1e-7 * v for a, b in seen):
                continue
            s1 = np.sqrt(b2 / q)
            P = f * np.array([s1, u * s1, v * s1])[:, None]
            R = frame(P) @ frame(X).T
            t = P[0] - R @ X[0]
            if np.all(np.isfinite(R)) and np.all(np.isfinite(t)):
                sols.append((R, t)); seen.append((u, v))
    return sols


def p3p_four_points(X, x, K):
    """cv::solvePnPRansac with exactly four points (modules/calib3d solvepnp.cpp: model_points = 4, SOLVEPNP_P3P, a single
    cv::solvePnP on all four, no RANSAC, no refinement): P3P on the first three points -- image points normalised as
    cv::undistortPoints stores them (f32) -- and the fourth picks the solution by its squared pixel reprojection error.
    Returns (rvec, tvec) or None.  Pinned against cv2 to 1e-5 (the f32 normalisation is what bounds it)."""
    X = np.asarray(X, np.float32).reshape(4, 3).astype(np.float64)
    x32 = np.asarray(x, np.float32).reshape(4, 2)
    K64 = np.asarray(K, np.float64)
    fx, fy, cx, cy = K64[0, 0], K64[1, 1], K64[0, 2], K64[1, 2]
    yn = undistort_normalize_f32(x32, K64).astype(np.float64)
    xp = x32.astype(np.float64)
    best = None
    for R, t in p3p_solutions(X[:3], yn[:3]):
        Xc = R @ X[3] + t
        e = (cx + fx * Xc[0] / Xc[2] - xp[3, 0]) ** 2 + (cy + fy * Xc[1] / Xc[2] - xp[3, 1]) ** 2
        if np.isfinite(e) and (best is None or e < best[0]):
            best = (e, R, t)
    if best is None:
        return None
    return rodrigues_inv(best[1]), best[2]


# ----------------------------------------------------------------------------- solvePnPRansac
def solve_pnp_ransac(X, x, K, rvec0, tvec0, iterations=500, reproj=0.5, confidence=0.999, trace=None,
                     model_fn=None):
    """cv::solvePnPRansac(..., useExtrinsicGuess=true, SOLVEPNP_ITERATIVE); n == 4 is the P3P case above, n == 5 a
    single unrefined EPnP.
    model_fn(Xs, xs, K) -> (rvec, tvec) defaults to the EPnP restatement."""
    X = np.asarray(X, np.float32).reshape(-1, 3)
    x = np.asarray(x, np.float32).reshape(-1, 2)
    K64 = np.asarray(K, np.float32).astype(np.float64)
    n = len(X)
    model_fn = model_fn or epnp
    if n == 4:
        m = p3p_four_points(X, x, K64)
        if m is None:
            return dict(ok=False, rvec=np.asarray(rvec0, np.float64), tvec=np.asarray(tvec0, np.float64),
                        inliers=np.zeros(0, np.int32), iters=0)
        return dict(ok=True, rvec=m[0], tvec=m[1], inliers=np.arange(4, dtype=np.int32), iters=0, model=m)
    assert n >= 5, "cv::solvePnPRansac needs at least four points"
    if n == 5:
        # n == model_points: no RANSAC, one EPnP solvePnP on all five, no refinement, all five inliers -- also when the
        # pose is not finite (five identical points: rvec 0, tvec nan)
        m = model_fn(X, x, K64)
        return dict(ok=True, rvec=m[0], tvec=m[1], inliers=np.arange(5, dtype=np.int32), iters=0, model=m)
    # RANSACPointSetRegistrator::run: CV_Assert(confidence > 0 && confidence < 1), then at least one iteration
    if not (0 < confidence < 1):
        raise ValueError(f"confidence={confidence} outside (0, 1): cv::solvePnPRansac asserts 0 < confidence < 1")
    rng = CvRNG(MASK64)
    thr = np.float32(np.float64(reproj) * np.float64(reproj))
    niters = max(int(iterations), 1)
    best_mask = None
    max_good = 0
    best_model = None
    it = 0
    while it < niters:
        idx = ransac_subset(rng, n, 5)
        rv, tv = model_fn(X[idx], x[idx], K64)
        err = reproj_err_f32(X, x, rv, tv, K64)
        mask = err <= thr
        good = int(mask.sum())
        if good > max(max_good, 4):
            best_mask = mask
            best_model = (rv, tv)
            max_good = good
            niters = ransac_update_num_iters(confidence, float(n - good) / n, 5, niters)
            if trace is not None:
                trace.append((it, good, niters))
        it += 1
    if best_mask is None:
        return dict(ok=False, rvec=np.asarray(rvec0, np.float64), tvec=np.asarray(tvec0, np.float64),
                    inliers=np.zeros(0, np.int32), iters=it)
    inl = np.nonzero(best_mask)[0].astype(np.int32)
    rv, tv = lm_refine(X[inl], x[inl], K64, rvec0, tvec0)
    return dict(ok=True, rvec=rv, tvec=tv, inliers=inl, iters=it, model=best_model)
