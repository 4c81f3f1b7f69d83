"""
oracle/essential_ref.py -- TEST INFRASTRUCTURE ONLY (never imported by the product path).

CPU restatement of the `mono_rotation = true` branch of the reference's trackingFrame2Frame
(reference src/visualOdometry.cpp:146-157):

    E = cv::findEssentialMat(pointsLeft_t0, pointsLeft_t1, focal, pp, cv::RANSAC, 0.999, 1.0, mask);
    cv::recoverPose(E, pointsLeft_t0, pointsLeft_t1, rotation, translation_mono, focal, pp, mask);

OpenCV's implementation (un-vendored third-party dependency, pinned here to 4.13.0; upstream
modules/calib3d/src/five-point.cpp + ptsetreg.cpp) is restated from its published algorithm:
Nister's five-point solver (null space of the 5x9 epipolar system, the ten cubic constraints in Nister's
monomial order, Gauss-Jordan, the 3x3 polynomial matrix B(z), its degree-10 determinant, one E per real
root), scored by the Sampson distance inside the same RANSAC point-set registrator solvePnPRansac uses
(cv::RNG(2^64-1), 5 distinct indices, `count > max(best, 4)`, adaptive iteration bound), then
decomposeEssentialMat + the four-way cheirality vote of recoverPose.

It is NOT operation-for-operation: the E candidates of a sample are a mathematical function of the five
correspondences, so any accurate solver produces the same set; tests pin this file against cv2 itself
(tests/test_oracle_essential.py: inlier masks and rotations on stress sets).
"""
import numpy as np

from .pnp_ref import CvRNG, MASK64, ransac_subset, ransac_update_num_iters

# Nister's monomial order of the constraint matrix columns
_MONO = [(3, 0, 0), (0, 3, 0), (2, 1, 0), (1, 2, 0), (2, 0, 1), (2, 0, 0), (0, 2, 1), (0, 2, 0), (1, 1, 1), (1, 1, 0),
         (1, 0, 2), (1, 0, 1), (1, 0, 0), (0, 1, 2), (0, 1, 1), (0, 1, 0), (0, 0, 3), (0, 0, 2), (0, 0, 1), (0, 0, 0)]
_MONO_IDX = {m: i for i, m in enumerate(_MONO)}


def _pmul(a, b):
    """product of two polynomials in (x, y, z) stored as {(i, j, k): coeff}"""
    out = {}
    for (i1, j1, k1), c1 in a.items():
        for (i2, j2, k2), c2 in b.items():
            key = (i1 + i2, j1 + j2, k1 + k2)
            out[key] = out.get(key, 0.0) + c1 * c2
    return out


def _padd(a, b, s=1.0):
    out = dict(a)
    for k, c in b.items():
        out[k] = out.get(k, 0.0) + s * c
    return out


def constraint_matrix(EE):
    """EE: 4 x 9 null-space basis (rows reshape to 3 x 3).  E(x, y, z) = x E0 + y E1 + z E2 + E3.
    Returns the 10 x 20 coefficient matrix of det(E) = 0 and 2 E E^T E - tr(E E^T) E = 0."""
    Eb = EE.reshape(4, 3, 3)
    var = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
    E = [[{var[b]: float(Eb[b, r, c]) for b in range(4)} for c in range(3)] for r in range(3)]
    rows = []
    # det(E)
    d = {}
    for (a, b, c), s in (((0, 1, 2), 1), ((1, 2, 0), 1), ((2, 0, 1), 1), ((2, 1, 0), -1), ((1, 0, 2), -1), ((0, 2, 1), -1)):
        d = _padd(d, _pmul(_pmul(E[0][a], E[1][b]), E[2][c]), s)
    rows.append(d)
    # EEt = E E^T
    EEt = [[{} for _ in range(3)] for _ in range(3)]
    for r in range(3):
        for c in range(3):
            acc = {}
            for k in range(3):
                acc = _padd(acc, _pmul(E[r][k], E[c][k]))
            EEt[r][c] = acc
    tr = _padd(_padd(EEt[0][0], EEt[1][1]), EEt[2][2])
    for r in range(3):
        for c in range(3):
            acc = {}
            for k in range(3):
                acc = _padd(acc, _pmul(EEt[r][k], E[k][c]), 2.0)
            acc = _padd(acc, _pmul(tr, E[r][c]), -1.0)
            rows.append(acc)
    A = np.zeros((10, 20))
    for i, p in enumerate(rows):
        for m, c in p.items():
            A[i, _MONO_IDX[m]] = c
    return A


def _poly1_mul(a, b):
    return np.convolve(a, b)


def five_point(q1, q2):
    """q1, q2: 5 x 2 normalised image points.  Returns the list of 3 x 3 essential matrices with q2^T E q1 = 0."""
    q1 = np.asarray(q1, np.float64); q2 = np.asarray(q2, np.float64)
    n = len(q1)
    # q2^T E q1 = 0 as a linear equation in the row-major entries of E
    Q = np.stack([q2[:, 0] * q1[:, 0], q2[:, 0] * q1[:, 1], q2[:, 0], q2[:, 1] * q1[:, 0], q2[:, 1] * q1[:, 1], q2[:, 1],
                  q1[:, 0], q1[:, 1], np.ones(n)], 1)
    _, _, Vt = np.linalg.svd(Q, full_matrices=True)
    EE = Vt[5:9]                                  # 4 x 9 null-space basis
    A = constraint_matrix(EE)
    try:
        A = np.linalg.solve(A[:, :10], A[:, 10:])
    except np.linalg.LinAlgError:
        return []
    # B(z): rows <e> - z <f> of the row pairs (4,5), (6,7), (8,9); columns [x: z^3..1 | y: z^3..1 | 1: z^4..1]
    B = np.zeros((3, 13))
    for i in range(3):
        r1, r2 = A[2 * i + 4], A[2 * i + 5]
        row1 = np.zeros(13); row2 = np.zeros(13)
        row1[1:4] = r1[0:3]; row1[5:8] = r1[3:6]; row1[9:13] = r1[6:10]
        row2[0:3] = r2[0:3]; row2[4:7] = r2[3:6]; row2[8:12] = r2[6:10]
        B[i] = row1 - row2
    P = [[B[i, 0:4], B[i, 4:8], B[i, 8:13]] for i in range(3)]       # polynomials in z, highest degree first
    det = np.zeros(11)
    for (a, b, c), s in (((0, 1, 2), 1), ((1, 2, 0), 1), ((2, 0, 1), 1), ((2, 1, 0), -1), ((1, 0, 2), -1), ((0, 2, 1), -1)):
        t = _poly1_mul(_poly1_mul(P[0][a], P[1][b]), P[2][c])
        det[11 - len(t):] += s * t
    roots = np.roots(det)
    out = []
    for z in roots:
        if abs(z.imag) > 1e-10:
            continue
        z = z.real
        zp = np.array([z ** 3, z ** 2, z, 1.0]); zq = np.array([z ** 4, z ** 3, z ** 2, z, 1.0])
        Bz = np.array([[P[i][0] @ zp, P[i][1] @ zp, P[i][2] @ zq] for i in range(3)])
        _, _, vt = np.linalg.svd(Bz)
        xy1 = vt[2]
        if abs(xy1[2]) < 1e-10:
            continue
        x, y = xy1[0] / xy1[2], xy1[1] / xy1[2]
        E = (x * EE[0] + y * EE[1] + z * EE[2] + EE[3]).reshape(3, 3)
        out.append(E)
    return out


def sampson_err_f32(E, q1, q2):
    """EMEstimatorCallback::computeError: squared Sampson distance, stored as float"""
    x1 = np.concatenate([q1, np.ones((len(q1), 1))], 1)
    x2 = np.concatenate([q2, np.ones((len(q2), 1))], 1)
    Ex1 = x1 @ E.T
    Etx2 = x2 @ E
    x2tEx1 = np.sum(x2 * Ex1, 1)
    den = Ex1[:, 0] ** 2 + Ex1[:, 1] ** 2 + Etx2[:, 0] ** 2 + Etx2[:, 1] ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        return (x2tEx1 * x2tEx1 / den).astype(np.float32)


def find_essential_mat(p1, p2, focal, pp, prob=0.999, threshold=1.0, max_iters=1000, trace=None):
    """cv::findEssentialMat(p1, p2, focal, pp, RANSAC, prob, threshold, mask) -> (E, mask, iterations).
    With exactly five points OpenCV runs no RANSAC: E is every candidate of one solve stacked (3k x 3, None for k = 0)
    and the mask is all ones."""
    p1 = np.asarray(p1, np.float32).astype(np.float64).reshape(-1, 2)
    p2 = np.asarray(p2, np.float32).astype(np.float64).reshape(-1, 2)
    n = len(p1)
    q1 = (p1 - np.array(pp)) / focal
    q2 = (p2 - np.array(pp)) / focal
    if n == 5:
        Es = five_point(q1, q2)
        return (np.vstack(Es) if Es else None), np.ones(n, bool), 0
    thr = threshold / focal                      # threshold /= (fx + fy) / 2
    t = np.float32(thr * thr)
    rng = CvRNG(MASK64)
    niters = max_iters
    best_E, best_mask, max_good = None, None, 0
    it = 0
    while it < niters:
        idx = ransac_subset(rng, n, 5)
        for E in five_point(q1[idx], q2[idx]):
            mask = sampson_err_f32(E, q1, q2) <= t
            good = int(mask.sum())
            if good > max(max_good, 4):
                best_E, best_mask, max_good = E, mask, good
                niters = ransac_update_num_iters(prob, float(n - good) / n, 5, niters)
                if trace is not None:
                    trace.append((it, good, niters))
        it += 1
    if best_E is None:
        return None, np.zeros(n, bool), it
    return best_E, best_mask, it


def _triangulate_f64(P0, P1, q1, q2):
    X = np.zeros((4, len(q1)))
    for i in range(len(q1)):
        A = np.stack([q1[i, 0] * P0[2] - P0[0], q1[i, 1] * P0[2] - P0[1], q2[i, 0] * P1[2] - P1[0], q2[i, 1] * P1[2] - P1[1]])
        _, _, vt = np.linalg.svd(A)
        X[:, i] = vt[3]
    return X


def recover_pose(E, p1, p2, focal, pp, mask, distance_thresh=50.0):
    """cv::recoverPose(E, p1, p2, R, t, focal, pp, mask) -> (R, t, mask_out, n_good)"""
    p1 = np.asarray(p1, np.float32).astype(np.float64).reshape(-1, 2)
    p2 = np.asarray(p2, np.float32).astype(np.float64).reshape(-1, 2)
    q1 = (p1 - np.array(pp)) / focal
    q2 = (p2 - np.array(pp)) / focal
    U, _, Vt = np.linalg.svd(E)
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(Vt) < 0:
        Vt = -Vt
    W = np.array([[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    R1 = U @ W @ Vt
    R2 = U @ W.T @ Vt
    t = U[:, 2]
    P0 = np.hstack([np.eye(3), np.zeros((3, 1))])
    cands = [(R1, t), (R2, t), (R1, -t), (R2, -t)]
    masks = []
    for R, tt in cands:
        P = np.hstack([R, tt.reshape(3, 1)])
        Q = _triangulate_f64(P0, P, q1, q2)
        m = (Q[2] * Q[3]) > 0
        with np.errstate(divide="ignore", invalid="ignore"):
            Q3 = Q[:3] / Q[3]
        m &= Q3[2] < distance_thresh
        Qc = P @ np.vstack([Q3, np.ones(Q.shape[1])])
        m &= Qc[2] > 0
        m &= Qc[2] < distance_thresh
        m &= np.asarray(mask, bool)
        masks.append(m)
    good = [int(m.sum()) for m in masks]
    if good[0] >= good[1] and good[0] >= good[2] and good[0] >= good[3]:
        k = 0
    elif good[1] >= good[0] and good[1] >= good[2] and good[1] >= good[3]:
        k = 1
    elif good[2] >= good[0] and good[2] >= good[1] and good[2] >= good[3]:
        k = 2
    else:
        k = 3
    return cands[k][0], cands[k][1], masks[k], good[k]


def mono_rotation(p_t0, p_t1, focal, pp):
    """The rotation the reference's mono branch leaves in `rotation` (reference src/visualOdometry.cpp:152-156); None
    where the reference aborts: no model, or (five points) a stack of several candidates, which recoverPose refuses."""
    E, mask, iters = find_essential_mat(p_t0, p_t1, focal, pp)
    if E is None or E.shape != (3, 3):
        return None, mask, iters
    R, t, m2, good = recover_pose(E, p_t0, p_t1, focal, pp, mask)
    return R, mask, iters
