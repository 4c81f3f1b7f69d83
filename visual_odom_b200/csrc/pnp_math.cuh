// pnp_math.cuh -- small dense fp64 linear algebra + EPnP + Rodrigues, host/device.
//
// Everything here follows OpenCV 4.13's arithmetic operation-for-operation (the algorithms the
// reference reaches through cv::solvePnPRansac / cv::triangulatePoints, reference
// src/visualOdometry.cpp:176-178, src/main.cpp:170): one-sided Jacobi SVD with OpenCV's scaled
// hypot and scalar sequential dot products, SVD back-substitution (cv::solve / cv::invert with
// DECOMP_SVD), sequential M^T M, EPnP with its Householder QR Gauss-Newton.  The 5-point EPnP
// kernel has a rank-10 12x12 Gram matrix whose two null-space left singular vectors are pure
// rounding noise, so the result is only reproducible if every operation rounds like the CPU
// build: compile with -fmad=false (no FMA contraction) -- visual_odom_b200/build.py does.
// Restated independently in oracle/pnp_ref.py (pinned bit-for-bit against cv2).
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define VO_HD __host__ __device__ __forceinline__
#define VO_HDN __host__ __device__
#else
#define VO_HD inline
#define VO_HDN
#endif

namespace vomath {

constexpr double kDblMin = 2.2250738585072014e-308;
constexpr double kDblEps = 2.220446049250313e-16;

// cv::RNG (multiply-with-carry)
struct Rng {
    uint64_t state;
    VO_HD explicit Rng(uint64_t s) : state(s ? s : 0xffffffffffffffffULL) {}
    VO_HD uint32_t next()
    {
        state = (uint64_t)(uint32_t)state * 4164903690ULL + (state >> 32);
        return (uint32_t)state;
    }
};

// cv::RANSACUpdateNumIters (ptsetreg.cpp)
VO_HDN inline int ransac_update_num_iters(double p, double ep, int model_points, int max_iters)
{
    p = fmax(p, 0.); p = fmin(p, 1.);
    ep = fmax(ep, 0.); ep = fmin(ep, 1.);
    double num = fmax(1. - p, kDblMin);
    double denom = 1. - pow(1. - ep, (double)model_points);
    if (denom < kDblMin) return 0;
    num = log(num);
    denom = log(denom);
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int)rint(num / denom);
}

VO_HD double cv_hypot(double a, double b)
{
    a = fabs(a); b = fabs(b);
    if (a > b) { b /= a; return a * sqrt(1 + b * b); }
    if (b > 0) { a /= b; return b * sqrt(1 + a * a); }
    return 0;
}

// JacobiSVDImpl_<double>: At is N rows x M (= A^T, row stride M), on exit rows of At are U^T
// (first n1 rows normalised), W singular values (descending), Vt N x N.
// WANT_V = false skips the accumulation of V (it never feeds back into At / W, so U^T and W are
// bit-identical either way); Vt may then be nullptr.
// The body is written once (JSVD_BODY) and instantiated with or without full unrolling of every loop over a compile-time
// extent.  Fully unrolled (the 4x4 of triangulate_dlt, one per thread), every index is a constant and At / W / Vt live in
// registers; the row swap of the sort is a compare per row rather than an index.  Larger systems keep plain loops:
// unrolled, the 12x12 and 6x6 instances made k_pnp_hypotheses spill several times more.  (A counted `#pragma unroll 4`
// does not help: it is applied after the arrays have been assigned to memory.)  Both forms do the same operations in the
// same order.
#define JSVD_BODY(JSVD_UNROLL)                                                                                              \
    const double eps = kDblEps * 10;                                                                                        \
    JSVD_UNROLL for (int i = 0; i < N; i++) {                                                                               \
        double sd = 0;                                                                                                      \
        JSVD_UNROLL for (int k = 0; k < M; k++) { double t = At[i * M + k]; sd += t * t; }                                  \
        W[i] = sd;                                                                                                          \
        if (WANT_V) {                                                                                                       \
            JSVD_UNROLL for (int k = 0; k < N; k++) Vt[i * N + k] = 0;                                                      \
            Vt[i * N + i] = 1;                                                                                              \
        }                                                                                                                   \
    }                                                                                                                       \
    const int max_iter = M > 30 ? M : 30;                                                                                   \
    for (int iter = 0; iter < max_iter; iter++) {                                                                           \
        bool changed = false;                                                                                               \
        JSVD_UNROLL for (int i = 0; i < N - 1; i++)                                                                         \
            JSVD_UNROLL for (int j = 0; j < N; j++) {      /* j = i + 1 .. N - 1 */                                         \
                if (j <= i) continue;                                                                                       \
                double* Ai = At + i * M; double* Aj = At + j * M;                                                           \
                double a = W[i], p = 0, b = W[j];                                                                           \
                JSVD_UNROLL for (int k = 0; k < M; k++) p += Ai[k] * Aj[k];                                                 \
                if (fabs(p) <= eps * sqrt(a * b)) continue;                                                                 \
                p *= 2;                                                                                                     \
                double beta = a - b, gamma = cv_hypot(p, beta), c, s;                                                       \
                if (beta < 0) {                                                                                             \
                    double delta = (gamma - beta) * 0.5;                                                                    \
                    s = sqrt(delta / gamma);                                                                                \
                    c = p / (gamma * s * 2);                                                                                \
                } else {                                                                                                    \
                    c = sqrt((gamma + beta) / (gamma * 2));                                                                 \
                    s = p / (gamma * c * 2);                                                                                \
                }                                                                                                           \
                a = b = 0;                                                                                                  \
                JSVD_UNROLL for (int k = 0; k < M; k++) {                                                                   \
                    double t0 = c * Ai[k] + s * Aj[k];                                                                      \
                    double t1 = -s * Ai[k] + c * Aj[k];                                                                     \
                    Ai[k] = t0; Aj[k] = t1;                                                                                 \
                    a += t0 * t0; b += t1 * t1;                                                                             \
                }                                                                                                           \
                W[i] = a; W[j] = b;                                                                                         \
                changed = true;                                                                                             \
                if (WANT_V) {                                                                                               \
                    double* Vi = Vt + i * N; double* Vj = Vt + j * N;                                                       \
                    JSVD_UNROLL for (int k = 0; k < N; k++) {                                                               \
                        double t0 = c * Vi[k] + s * Vj[k];                                                                  \
                        double t1 = -s * Vi[k] + c * Vj[k];                                                                 \
                        Vi[k] = t0; Vj[k] = t1;                                                                             \
                    }                                                                                                       \
                }                                                                                                           \
            }                                                                                                               \
        if (!changed) break;                                                                                                \
    }                                                                                                                       \
    JSVD_UNROLL for (int i = 0; i < N; i++) {                                                                               \
        double sd = 0;                                                                                                      \
        JSVD_UNROLL for (int k = 0; k < M; k++) { double t = At[i * M + k]; sd += t * t; }                                  \
        W[i] = sqrt(sd);                                                                                                    \
    }                                                                                                                       \
    /* selection sort (first maximum wins); the swap partner is found by comparison, never used as an index */              \
    JSVD_UNROLL for (int i = 0; i < N - 1; i++) {                                                                           \
        int j = i;                                                                                                          \
        double wj = W[i];                                                                                                   \
        JSVD_UNROLL for (int k = 0; k < N; k++)                                                                             \
            if (k > i && wj < W[k]) { wj = W[k]; j = k; }                                                                   \
        JSVD_UNROLL for (int q = 0; q < N; q++) {                                                                           \
            if (q <= i || q != j) continue;                                                                                 \
            double t = W[i]; W[i] = W[q]; W[q] = t;                                                                         \
            JSVD_UNROLL for (int k = 0; k < M; k++) { t = At[i * M + k]; At[i * M + k] = At[q * M + k]; At[q * M + k] = t; } \
            if (WANT_V) JSVD_UNROLL for (int k = 0; k < N; k++) { t = Vt[i * N + k]; Vt[i * N + k] = Vt[q * N + k]; Vt[q * N + k] = t; } \
        }                                                                                                                   \
    }                                                                                                                       \
    Rng rng(0x12345678);                                                                                                    \
    JSVD_UNROLL for (int i = 0; i < n1; i++) {                                                                              \
        double sd = i < N ? W[i] : 0;                                                                                       \
        for (int ii = 0; ii < 100 && sd <= kDblMin; ii++) {                                                                 \
            /* exactly-zero singular value: random +-1/M vector, Gram-Schmidt against previous rows */                      \
            const double val0 = 1. / M;                                                                                     \
            JSVD_UNROLL for (int k = 0; k < M; k++) At[i * M + k] = (rng.next() & 256) != 0 ? val0 : -val0;                 \
            for (int it = 0; it < 2; it++)                                                                                  \
                JSVD_UNROLL for (int j = 0; j < N; j++) {                                                                   \
                    if (j >= i) continue;                                                                                   \
                    sd = 0;                                                                                                 \
                    JSVD_UNROLL for (int k = 0; k < M; k++) sd += At[i * M + k] * At[j * M + k];                            \
                    double asum = 0;                                                                                        \
                    JSVD_UNROLL for (int k = 0; k < M; k++) {                                                               \
                        double t = At[i * M + k] - sd * At[j * M + k];                                                      \
                        At[i * M + k] = t;                                                                                  \
                        asum += fabs(t);                                                                                    \
                    }                                                                                                       \
                    asum = asum > eps * 100 ? 1 / asum : 0;                                                                 \
                    JSVD_UNROLL for (int k = 0; k < M; k++) At[i * M + k] *= asum;                                          \
                }                                                                                                           \
            sd = 0;                                                                                                         \
            JSVD_UNROLL for (int k = 0; k < M; k++) { double t = At[i * M + k]; sd += t * t; }                              \
            sd = sqrt(sd);                                                                                                  \
        }                                                                                                                   \
        const double s = sd > kDblMin ? 1 / sd : 0.;                                                                        \
        JSVD_UNROLL for (int k = 0; k < M; k++) At[i * M + k] *= s;                                                         \
    }                                                                                                                       \

#if defined(__CUDA_ARCH__)
#define JSVD_FULL_UNROLL _Pragma("unroll")
#else
#define JSVD_FULL_UNROLL
#endif

template <int M, int N, bool WANT_V = true>
VO_HDN void jacobi_svd_t(double* At, double* W, double* Vt, int n1)
{
    if constexpr (M == 4 && N == 4) {
        JSVD_BODY(JSVD_FULL_UNROLL)
    } else {
        JSVD_BODY()
    }
}
#undef JSVD_FULL_UNROLL
#undef JSVD_BODY

// cv::solve(A (M x N row-major), b, x, DECOMP_SVD), one right-hand side
template <int M, int N>
VO_HDN void solve_svd(const double* A, const double* b, double* x)
{
    double At[N * M], W[N], Vt[N * N];
    for (int i = 0; i < M; i++)
        for (int j = 0; j < N; j++) At[j * M + i] = A[i * N + j];
    jacobi_svd_t<M, N>(At, W, Vt, N);
    double threshold = 0;
    for (int i = 0; i < N; i++) threshold += W[i];
    threshold *= kDblEps * 2;
    for (int j = 0; j < N; j++) x[j] = 0;
    for (int i = 0; i < N; i++) {
        double wi = W[i];
        if (fabs(wi) <= threshold) continue;
        wi = 1 / wi;
        double s = 0;
        for (int j = 0; j < M; j++) s += At[i * M + j] * b[j];
        s *= wi;
        for (int j = 0; j < N; j++) x[j] = x[j] + s * Vt[i * N + j];
    }
}

// The same one-sided Jacobi with the column count N a RUN-TIME value (N <= NMAX): identical arithmetic and order as
// jacobi_svd_t<M, N>, so lanes of one warp can solve systems of different widths in lockstep (EPnP's three beta
// approximations are 6x4, 6x3 and 6x5 least-squares problems).  Rows of At / Vt are N-strided exactly like the template.
template <int M, int NMAX>
VO_HDN void jacobi_svd_rt(double* At, double* W, double* Vt, int N)
{
    const double eps = kDblEps * 10;
    for (int i = 0; i < N; i++) {
        double sd = 0;
        for (int k = 0; k < M; k++) { double t = At[i * M + k]; sd += t * t; }
        W[i] = sd;
        for (int k = 0; k < N; k++) Vt[i * N + k] = 0;
        Vt[i * N + i] = 1;
    }
    const int max_iter = M > 30 ? M : 30;
    for (int iter = 0; iter < max_iter; iter++) {
        bool changed = false;
        for (int i = 0; i < N - 1; i++)
            for (int j = i + 1; j < N; j++) {
                double* Ai = At + i * M; double* Aj = At + j * M;
                double a = W[i], p = 0, b = W[j];
                for (int k = 0; k < M; k++) p += Ai[k] * Aj[k];
                if (fabs(p) <= eps * sqrt(a * b)) continue;
                p *= 2;
                double beta = a - b, gamma = cv_hypot(p, beta), c, s;
                if (beta < 0) {
                    double delta = (gamma - beta) * 0.5;
                    s = sqrt(delta / gamma);
                    c = p / (gamma * s * 2);
                } else {
                    c = sqrt((gamma + beta) / (gamma * 2));
                    s = p / (gamma * c * 2);
                }
                a = b = 0;
                for (int k = 0; k < M; k++) {
                    double t0 = c * Ai[k] + s * Aj[k];
                    double t1 = -s * Ai[k] + c * Aj[k];
                    Ai[k] = t0; Aj[k] = t1;
                    a += t0 * t0; b += t1 * t1;
                }
                W[i] = a; W[j] = b;
                changed = true;
                double* Vi = Vt + i * N; double* Vj = Vt + j * N;
                for (int k = 0; k < N; k++) {
                    double t0 = c * Vi[k] + s * Vj[k];
                    double t1 = -s * Vi[k] + c * Vj[k];
                    Vi[k] = t0; Vj[k] = t1;
                }
            }
        if (!changed) break;
    }
    for (int i = 0; i < N; i++) {
        double sd = 0;
        for (int k = 0; k < M; k++) { double t = At[i * M + k]; sd += t * t; }
        W[i] = sqrt(sd);
    }
    for (int i = 0; i < N - 1; i++) {
        int j = i;
        for (int k = i + 1; k < N; k++)
            if (W[j] < W[k]) j = k;
        if (i != j) {
            double t = W[i]; W[i] = W[j]; W[j] = t;
            for (int k = 0; k < M; k++) { t = At[i * M + k]; At[i * M + k] = At[j * M + k]; At[j * M + k] = t; }
            for (int k = 0; k < N; k++) { t = Vt[i * N + k]; Vt[i * N + k] = Vt[j * N + k]; Vt[j * N + k] = t; }
        }
    }
    Rng rng(0x12345678);
    for (int i = 0; i < N; i++) {
        double sd = W[i];
        for (int ii = 0; ii < 100 && sd <= kDblMin; ii++) {
            const double val0 = 1. / M;
            for (int k = 0; k < M; k++) At[i * M + k] = (rng.next() & 256) != 0 ? val0 : -val0;
            for (int it = 0; it < 2; it++)
                for (int j = 0; j < i; j++) {
                    sd = 0;
                    for (int k = 0; k < M; k++) sd += At[i * M + k] * At[j * M + k];
                    double asum = 0;
                    for (int k = 0; k < M; k++) {
                        double t = At[i * M + k] - sd * At[j * M + k];
                        At[i * M + k] = t;
                        asum += fabs(t);
                    }
                    asum = asum > eps * 100 ? 1 / asum : 0;
                    for (int k = 0; k < M; k++) At[i * M + k] *= asum;
                }
            sd = 0;
            for (int k = 0; k < M; k++) { double t = At[i * M + k]; sd += t * t; }
            sd = sqrt(sd);
        }
        const double s = sd > kDblMin ? 1 / sd : 0.;
        for (int k = 0; k < M; k++) At[i * M + k] *= s;
    }
}

// cv::solve(A (M x N row-major), b, x, DECOMP_SVD) with run-time N <= NMAX
template <int M, int NMAX>
VO_HDN void solve_svd_rt(const double* A, const double* b, double* x, int N)
{
    double At[NMAX * M], W[NMAX], Vt[NMAX * NMAX];
    for (int i = 0; i < M; i++)
        for (int j = 0; j < N; j++) At[j * M + i] = A[i * N + j];
    jacobi_svd_rt<M, NMAX>(At, W, Vt, N);
    double threshold = 0;
    for (int i = 0; i < N; i++) threshold += W[i];
    threshold *= kDblEps * 2;
    for (int j = 0; j < N; j++) x[j] = 0;
    for (int i = 0; i < N; i++) {
        double wi = W[i];
        if (fabs(wi) <= threshold) continue;
        wi = 1 / wi;
        double s = 0;
        for (int j = 0; j < M; j++) s += At[i * M + j] * b[j];
        s *= wi;
        for (int j = 0; j < N; j++) x[j] = x[j] + s * Vt[i * N + j];
    }
}

// The step of CvLevMarq: (JtJ with its diagonal scaled by 1 + lambda) dx = JtErr, JtJ 6x6 row-major symmetric.
// OpenCV solves this system with cv::solve(DECOMP_SVD).  A Cholesky factorisation is used instead while the damped
// matrix is positive definite: a few hundred flops rather than a Jacobi SVD on one thread, and a solution whose backward
// error is as small (tests/test_oracle_lm_refine.py checks it against OpenCV's SVD solve on the host;
// tests/test_gpu_pnp_refine.py pins the refined pose to cv2 at 1e-8).  A matrix
// that is not positive definite in floating point (rank-deficient normal equations) takes OpenCV's own SVD solve, so
// there the step is OpenCV's bit for bit.  Returns true when the Cholesky path was taken.
VO_HD bool lm_solve6(const double* JtJ, const double* JtErr, double lambda, double* dx)
{
    double A[36], y[6];
    for (int k = 0; k < 36; k++) A[k] = JtJ[k];
    for (int k = 0; k < 6; k++) A[k * 7] *= 1. + lambda;
    bool spd = true;
    for (int j = 0; j < 6 && spd; j++) {
        double d = A[j * 7];
        for (int k = 0; k < j; k++) d -= A[j * 6 + k] * A[j * 6 + k];
        if (!(d > 0)) { spd = false; break; }
        d = sqrt(d);
        A[j * 7] = d;
        for (int i = j + 1; i < 6; i++) {
            double v = A[i * 6 + j];
            for (int k = 0; k < j; k++) v -= A[i * 6 + k] * A[j * 6 + k];
            A[i * 6 + j] = v / d;
        }
    }
    if (spd) {
        for (int i = 0; i < 6; i++) { double v = JtErr[i]; for (int k = 0; k < i; k++) v -= A[i * 6 + k] * y[k]; y[i] = v / A[i * 7]; }
        for (int i = 5; i >= 0; i--) { double v = y[i]; for (int k = i + 1; k < 6; k++) v -= A[k * 6 + i] * dx[k]; dx[i] = v / A[i * 7]; }
    } else {
        for (int k = 0; k < 36; k++) A[k] = JtJ[k];
        for (int k = 0; k < 6; k++) A[k * 7] *= 1. + lambda;
        solve_svd<6, 6>(A, JtErr, dx);
    }
    return spd;
}

// cv::invert(A 3x3, Ainv, DECOMP_SVD)
VO_HDN inline void invert3_svd(const double* A, double* Ainv)
{
    double At[9], W[3], Vt[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) At[j * 3 + i] = A[i * 3 + j];
    jacobi_svd_t<3, 3>(At, W, Vt, 3);
    double threshold = (W[0] + W[1] + W[2]) * (kDblEps * 2);
    for (int k = 0; k < 9; k++) Ainv[k] = 0;
    for (int i = 0; i < 3; i++) {
        double wi = W[i];
        if (fabs(wi) <= threshold) continue;
        wi = 1 / wi;
        double buf[3];
        for (int j = 0; j < 3; j++) buf[j] = At[i * 3 + j] * wi;
        for (int r = 0; r < 3; r++) {
            const double s = Vt[i * 3 + r];
            for (int j = 0; j < 3; j++) Ainv[r * 3 + j] = Ainv[r * 3 + j] + s * buf[j];
        }
    }
}

// cv::SVD::compute(A 3x3) -> w, u (3x3), vt
VO_HDN inline void svd3(const double* A, double* w, double* u, double* vt)
{
    double At[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) At[j * 3 + i] = A[i * 3 + j];
    jacobi_svd_t<3, 3>(At, w, vt, 3);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) u[i * 3 + j] = At[j * 3 + i];
}

VO_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// cv::Rodrigues: rotation vector -> matrix
VO_HDN inline void rodrigues_fwd(const double* r, double* R)
{
    double rx = r[0], ry = r[1], rz = r[2];
    const double theta = sqrt(rx * rx + ry * ry + rz * rz);
    if (theta < kDblEps) {
        for (int k = 0; k < 9; k++) R[k] = (k % 4 == 0) ? 1. : 0.;
        return;
    }
    const double c = cos(theta), s = sin(theta), c1 = 1. - c;
    const double itheta = theta ? 1. / theta : 0.;
    rx *= itheta; ry *= itheta; rz *= itheta;
    const double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
    const double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
    for (int k = 0; k < 9; k++) R[k] = c * ((k % 4 == 0) ? 1. : 0.) + c1 * rrt[k] + s * r_x[k];
}

// cv::Rodrigues: matrix -> rotation vector.  A matrix with an entry outside [-100, 100) or non-finite gives the zero
// vector (OpenCV's checkRange guard: a degenerate EPnP pose, e.g. five identical points, comes back as rvec = 0)
VO_HDN inline void rodrigues_inv(const double* Rin, double* r)
{
    for (int k = 0; k < 9; k++)
        if (!(Rin[k] >= -100. && Rin[k] < 100.)) { r[0] = r[1] = r[2] = 0.; return; }
    double w[3], U[9], Vt[9], R[9];
    svd3(Rin, w, U, Vt);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += U[i * 3 + k] * Vt[k * 3 + j];
            R[i * 3 + j] = s;
        }
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1) * 0.5;
    c = c > 1. ? 1. : c < -1. ? -1. : c;
    double theta = acos(c);
    if (s < 1e-5) {
        if (c > 0) { r[0] = r[1] = r[2] = 0; return; }
        double t = (R[0] + 1) * 0.5;
        rx = sqrt(t > 0. ? t : 0.);
        t = (R[4] + 1) * 0.5;
        ry = sqrt(t > 0. ? t : 0.) * (R[1] < 0 ? -1. : 1.);
        t = (R[8] + 1) * 0.5;
        rz = sqrt(t > 0. ? t : 0.) * (R[2] < 0 ? -1. : 1.);
        if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && (R[5] > 0) != (ry * rz > 0)) rz = -rz;
        theta /= sqrt(rx * rx + ry * ry + rz * rz);
        r[0] = rx * theta; r[1] = ry * theta; r[2] = rz * theta;
        return;
    }
    double vth = 1 / (2 * s);
    vth *= theta;
    r[0] = rx * vth; r[1] = ry * vth; r[2] = rz * vth;
}

// epnp::qr_solve for the 6x4 Gauss-Newton system (with its off-by-one column scan); returns
// false when a column is exactly zero (OpenCV then leaves x untouched).
VO_HDN inline bool qr_solve_6x4(double* A, double* b, double* X)
{
    const int nr = 6, nc = 4;
    double A1[6], A2[6];
    for (int k = 0; k < nc; k++) {
        const int kk = k * nc + k;
        double eta = fabs(A[kk]);
        int p = kk;
        for (int i = k + 1; i < nr; i++) {
            const double elt = fabs(A[p]);
            if (eta < elt) eta = elt;
            p += nc;
        }
        if (eta == 0) return false;
        const double inv_eta = 1. / eta;
        double sum2 = 0;
        p = kk;
        for (int i = k; i < nr; i++) { A[p] *= inv_eta; sum2 += A[p] * A[p]; p += nc; }
        double sigma = sqrt(sum2);
        if (A[kk] < 0) sigma = -sigma;
        A[kk] += sigma;
        A1[k] = sigma * A[kk];
        A2[k] = -eta * sigma;
        for (int j = k + 1; j < nc; j++) {
            p = kk;
            double sum = 0;
            for (int i = k; i < nr; i++) { sum += A[p] * A[p + j - k]; p += nc; }
            const double tau = sum / A1[k];
            p = kk;
            for (int i = k; i < nr; i++) { A[p + j - k] -= tau * A[p]; p += nc; }
        }
    }
    for (int j = 0; j < nc; j++) {
        const int jj = j * nc + j;
        int p = jj;
        double tau = 0;
        for (int i = j; i < nr; i++) { tau += A[p] * b[i]; p += nc; }
        tau /= A1[j];
        p = jj;
        for (int i = j; i < nr; i++) { b[i] -= tau * A[p]; p += nc; }
    }
    X[nc - 1] = b[nc - 1] / A2[nc - 1];
    for (int i = nc - 2; i >= 0; i--) {
        double sum = 0;
        for (int j = i + 1; j < nc; j++) sum += A[i * nc + j] * X[j];
        X[i] = (b[i] - sum) / A2[i];
    }
    return true;
}

// cv::solvePnP(..., SOLVEPNP_EPNP) on exactly 5 correspondences, zero distortion, in three stages so
// that the middle one (the 12x12 Jacobi SVD, 3/4 of the work) can be replaced by the warp-cooperative
// version in pnp.cu:  epnp5_front -> M^T M ;  SVD ;  epnp5_back(left singular vectors 11, 10, 9, 8).
//   Xw[5][3] object points (float inputs widened to double), uv[5][2] pixel coordinates (float),
//   fu, fv, uc, vc intrinsics (float values widened to double).  Out: rvec[3], tvec[3], R[9].
struct Epnp5State {
    double X[5][3], us[5][2], cws[4][3], al[5][4];
    double fu, fv, uc, vc;
};

VO_HDN inline void epnp5_front(const float* Xw_f, const float* uv_f, double fu, double fv, double uc, double vc,
                               Epnp5State& st, double* MtM /* 144, symmetric */)
{
    st.fu = fu; st.fv = fv; st.uc = uc; st.vc = vc;

    const int n = 5;
    double (&X)[5][3] = st.X; double (&us)[5][2] = st.us;
    for (int i = 0; i < n; i++) {
        for (int j = 0; j < 3; j++) X[i][j] = (double)Xw_f[3 * i + j];
        // undistortPoints (zero distortion): normalised coordinate in f64, STORED AS FLOAT
        const double ifx = 1. / fu, ify = 1. / fv;
        const float xn = (float)(((double)uv_f[2 * i] - uc) * ifx);
        const float yn = (float)(((double)uv_f[2 * i + 1] - vc) * ify);
        us[i][0] = (double)xn * fu + uc;
        us[i][1] = (double)yn * fv + vc;
    }
    // choose_control_points
    double (&cws)[4][3] = st.cws;
    for (int j = 0; j < 3; j++) cws[0][j] = 0;
    for (int i = 0; i < n; i++)
        for (int j = 0; j < 3; j++) cws[0][j] += X[i][j];
    for (int j = 0; j < 3; j++) cws[0][j] /= n;
    {
        double pw0[5][3], G[9], dc[3], At[9];
        for (int i = 0; i < n; i++)
            for (int j = 0; j < 3; j++) pw0[i][j] = X[i][j] - cws[0][j];
        for (int i = 0; i < 3; i++)
            for (int j = i; j < 3; j++) {
                double s = 0;
                for (int k = 0; k < n; k++) s += pw0[k][i] * pw0[k][j];
                G[i * 3 + j] = s; G[j * 3 + i] = s;
            }
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) At[j * 3 + i] = G[i * 3 + j];
        jacobi_svd_t<3, 3, false>(At, dc, nullptr, 3);         // rows of At = U^T = uct (V is not needed)
        for (int i = 1; i < 4; i++) {
            const double k = sqrt(dc[i - 1] / n);
            for (int j = 0; j < 3; j++) cws[i][j] = cws[0][j] + k * At[(i - 1) * 3 + j];
        }
    }
    // compute_barycentric_coordinates
    double (&al)[5][4] = st.al;
    {
        double cc[9], ci[9];
        for (int i = 0; i < 3; i++)
            for (int j = 1; j < 4; j++) cc[3 * i + j - 1] = cws[j][i] - cws[0][i];
        invert3_svd(cc, ci);
        for (int i = 0; i < n; i++) {
            for (int j = 0; j < 3; j++)
                al[i][1 + j] = ci[3 * j] * (X[i][0] - cws[0][0]) + ci[3 * j + 1] * (X[i][1] - cws[0][1]) +
                               ci[3 * j + 2] * (X[i][2] - cws[0][2]);
            al[i][0] = 1.0 - al[i][1] - al[i][2] - al[i][3];
        }
    }
    // M (10 x 12) and its Gram matrix (cv::mulTransposed: sequential sums over the rows)
    double M[10 * 12];
    for (int k = 0; k < 120; k++) M[k] = 0;
    for (int i = 0; i < n; i++)
        for (int j = 0; j < 4; j++) {
            M[(2 * i) * 12 + 3 * j] = al[i][j] * fu;
            M[(2 * i) * 12 + 3 * j + 2] = al[i][j] * (uc - us[i][0]);
            M[(2 * i + 1) * 12 + 3 * j + 1] = al[i][j] * fv;
            M[(2 * i + 1) * 12 + 3 * j + 2] = al[i][j] * (vc - us[i][1]);
        }
    for (int i = 0; i < 12; i++)
        for (int j = i; j < 12; j++) {
            double s = 0;
            for (int k = 0; k < 10; k++) s += M[k * 12 + i] * M[k * 12 + j];
            MtM[i * 12 + j] = s; MtM[j * 12 + i] = s;
        }
}

// v0..v3: rows 11, 10, 9, 8 of U^T of the SVD of M^T M (12 doubles each)
// One of EPnP's three beta initialisations (approx = 1: betas from [B11 B12 B13 B14], 2: [B11 B12 B22], 3: [B11 B12 B22 B13
// B23]) -> Gauss-Newton -> R, t and the mean reprojection error of the 5 points.  The three are independent, so the
// hypothesis kernel runs them on three lanes in lockstep (run-time system width) and picks like the reference does.
// Always inlined.  Compiled as a separate (__noinline__) device function by NVVM at -O3 (CUDA 12.9, compute_90a), the beta
// least-squares solve below (solve_svd_rt) returned NaN on an H100 although L and rho going into it were exact, and ptxas at
// -O0 gave the same NaN.  No undefined behaviour was found in this source and the failing PTX instruction has not been
// isolated, so the cause is unconfirmed: do not make this function out-of-line again without rerunning the GPU PnP tests.
VO_HD void epnp5_back_one(const Epnp5State& st, const double* v0, const double* v1, const double* v2, const double* v3,
                                  int approx, double* R, double* t, double* err_out)
{

    const int n = 5;
    const double (&X)[5][3] = st.X; const double (&us)[5][2] = st.us;
    const double (&cws)[4][3] = st.cws; const double (&al)[5][4] = st.al;
    const double fu = st.fu, fv = st.fv, uc = st.uc, vc = st.vc;
    const double* v[4] = {v0, v1, v2, v3};
    double L[6][10], rho[6];
    {
        double dv[4][6][3];
        for (int i = 0; i < 4; i++) {
            int a = 0, b = 1;
            for (int j = 0; j < 6; j++) {
                dv[i][j][0] = v[i][3 * a] - v[i][3 * b];
                dv[i][j][1] = v[i][3 * a + 1] - v[i][3 * b + 1];
                dv[i][j][2] = v[i][3 * a + 2] - v[i][3 * b + 2];
                b++;
                if (b > 3) { a++; b = a + 1; }
            }
        }
        for (int i = 0; i < 6; i++) {
            L[i][0] = dot3(dv[0][i], dv[0][i]);
            L[i][1] = 2.0 * dot3(dv[0][i], dv[1][i]);
            L[i][2] = dot3(dv[1][i], dv[1][i]);
            L[i][3] = 2.0 * dot3(dv[0][i], dv[2][i]);
            L[i][4] = 2.0 * dot3(dv[1][i], dv[2][i]);
            L[i][5] = dot3(dv[2][i], dv[2][i]);
            L[i][6] = 2.0 * dot3(dv[0][i], dv[3][i]);
            L[i][7] = 2.0 * dot3(dv[1][i], dv[3][i]);
            L[i][8] = 2.0 * dot3(dv[2][i], dv[3][i]);
            L[i][9] = dot3(dv[3][i], dv[3][i]);
        }
        int a = 0, b = 1;
        for (int j = 0; j < 6; j++) {
            const double d0 = cws[a][0] - cws[b][0], d1 = cws[a][1] - cws[b][1], d2 = cws[a][2] - cws[b][2];
            rho[j] = d0 * d0 + d1 * d1 + d2 * d2;
            b++;
            if (b > 3) { a++; b = a + 1; }
        }
    }
    double x_last[4] = {0, 0, 0, 0};
    {
        double be[4];
        {
            // the beta estimate: least squares on the first ncol columns of L (in the order B11 B12 B13 B14 for approx 1)
            const int ncol = approx == 1 ? 4 : (approx == 2 ? 3 : 5);
            double A[30], bs[5] = {0, 0, 0, 0, 0};
            for (int i = 0; i < 6; i++) {
                if (approx == 1) { A[i * 4] = L[i][0]; A[i * 4 + 1] = L[i][1]; A[i * 4 + 2] = L[i][3]; A[i * 4 + 3] = L[i][6]; }
                else for (int c = 0; c < ncol; c++) A[i * ncol + c] = L[i][c];
            }
            solve_svd_rt<6, 5>(A, rho, bs, ncol);
            if (approx == 1) {
                if (bs[0] < 0) { be[0] = sqrt(-bs[0]); be[1] = -bs[1] / be[0]; be[2] = -bs[2] / be[0]; be[3] = -bs[3] / be[0]; }
                else { be[0] = sqrt(bs[0]); be[1] = bs[1] / be[0]; be[2] = bs[2] / be[0]; be[3] = bs[3] / be[0]; }
            } else {
                if (bs[0] < 0) { be[0] = sqrt(-bs[0]); be[1] = (bs[2] < 0) ? sqrt(-bs[2]) : 0.0; }
                else { be[0] = sqrt(bs[0]); be[1] = (bs[2] > 0) ? sqrt(bs[2]) : 0.0; }
                if (bs[1] < 0) be[0] = -be[0];
                be[2] = approx == 3 ? bs[3] / be[0] : 0.0;
                be[3] = 0.0;
            }
        }
        // gauss_newton: 5 iterations
        x_last[0] = x_last[1] = x_last[2] = x_last[3] = 0;
        for (int it = 0; it < 5; it++) {
            double A[24], b[6];
            for (int i = 0; i < 6; i++) {
                const double* r = L[i];
                A[i * 4 + 0] = 2 * r[0] * be[0] + r[1] * be[1] + r[3] * be[2] + r[6] * be[3];
                A[i * 4 + 1] = r[1] * be[0] + 2 * r[2] * be[1] + r[4] * be[2] + r[7] * be[3];
                A[i * 4 + 2] = r[3] * be[0] + r[4] * be[1] + 2 * r[5] * be[2] + r[8] * be[3];
                A[i * 4 + 3] = r[6] * be[0] + r[7] * be[1] + r[8] * be[2] + 2 * r[9] * be[3];
                b[i] = rho[i] - (r[0] * be[0] * be[0] + r[1] * be[0] * be[1] + r[2] * be[1] * be[1] +
                                 r[3] * be[0] * be[2] + r[4] * be[1] * be[2] + r[5] * be[2] * be[2] +
                                 r[6] * be[0] * be[3] + r[7] * be[1] * be[3] + r[8] * be[2] * be[3] +
                                 r[9] * be[3] * be[3]);
            }
            qr_solve_6x4(A, b, x_last);
            for (int i = 0; i < 4; i++) be[i] += x_last[i];
        }
        // compute_R_and_t
        double ccs[4][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
        for (int i = 0; i < 4; i++)
            for (int j = 0; j < 4; j++)
                for (int k = 0; k < 3; k++) ccs[j][k] += be[i] * v[i][3 * j + k];
        double pcs[5][3];
        for (int i = 0; i < n; i++)
            for (int j = 0; j < 3; j++)
                pcs[i][j] = al[i][0] * ccs[0][j] + al[i][1] * ccs[1][j] + al[i][2] * ccs[2][j] + al[i][3] * ccs[3][j];
        if (pcs[0][2] < 0.0)
            for (int i = 0; i < n; i++)
                for (int j = 0; j < 3; j++) pcs[i][j] = -pcs[i][j];
        double pc0[3] = {0, 0, 0}, pw0[3] = {0, 0, 0};
        for (int i = 0; i < n; i++)
            for (int j = 0; j < 3; j++) { pc0[j] += pcs[i][j]; pw0[j] += X[i][j]; }
        for (int j = 0; j < 3; j++) { pc0[j] /= n; pw0[j] /= n; }
        double abt[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (int i = 0; i < n; i++)
            for (int j = 0; j < 3; j++) {
                abt[3 * j] += (pcs[i][j] - pc0[j]) * (X[i][0] - pw0[0]);
                abt[3 * j + 1] += (pcs[i][j] - pc0[j]) * (X[i][1] - pw0[1]);
                abt[3 * j + 2] += (pcs[i][j] - pc0[j]) * (X[i][2] - pw0[2]);
            }
        double w3[3], U[9], Vt3[9];
        svd3(abt, w3, U, Vt3);
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++)      // dot(abt_u row i, abt_v row j), abt_v = V (not V^T)
                R[i * 3 + j] = U[i * 3] * Vt3[j] + U[i * 3 + 1] * Vt3[3 + j] + U[i * 3 + 2] * Vt3[6 + j];
        const double det = R[0] * R[4] * R[8] + R[1] * R[5] * R[6] + R[2] * R[3] * R[7] -
                           R[2] * R[4] * R[6] - R[1] * R[3] * R[8] - R[0] * R[5] * R[7];
        if (det < 0) { R[6] = -R[6]; R[7] = -R[7]; R[8] = -R[8]; }
        t[0] = pc0[0] - dot3(R, pw0);
        t[1] = pc0[1] - dot3(R + 3, pw0);
        t[2] = pc0[2] - dot3(R + 6, pw0);
        double sum2 = 0;
        for (int i = 0; i < n; i++) {
            const double Xc = dot3(R, X[i]) + t[0], Yc = dot3(R + 3, X[i]) + t[1];
            const double inv_Zc = 1.0 / (dot3(R + 6, X[i]) + t[2]);
            const double ue = uc + fu * Xc * inv_Zc, ve = vc + fv * Yc * inv_Zc;
            const double u = us[i][0], vv = us[i][1];
            sum2 += sqrt((u - ue) * (u - ue) + (vv - ve) * (vv - ve));
        }
        *err_out = sum2 / n;
    }
}

VO_HDN inline void epnp5_back(const Epnp5State& st, const double* v0, const double* v1, const double* v2, const double* v3,
                              double* rvec, double* tvec, double* Rout)
{
    double best_err = 0, best_R[9], best_t[3];
    for (int approx = 1; approx <= 3; approx++) {
        double R[9], t[3], err;
        epnp5_back_one(st, v0, v1, v2, v3, approx, R, t, &err);
        // N = 2 if err2 < err1; N = 3 if err3 < err[N]
        if (approx == 1 || err < best_err) {
            best_err = err;
            for (int k = 0; k < 9; k++) best_R[k] = R[k];
            for (int k = 0; k < 3; k++) best_t[k] = t[k];
        }
    }
    rodrigues_inv(best_R, rvec);
    for (int k = 0; k < 3; k++) tvec[k] = best_t[k];
    // PnPRansacCallback::computeError -> projectPoints(rvec) converts back with Rodrigues
    rodrigues_fwd(rvec, Rout);
}


VO_HDN inline void epnp5(const float* Xw_f, const float* uv_f, double fu, double fv, double uc, double vc,
                         double* rvec, double* tvec, double* Rout)
{
    Epnp5State st;
    double ut[144], W[12];
    epnp5_front(Xw_f, uv_f, fu, fv, uc, vc, st, ut);                 // symmetric: A^T == A
    jacobi_svd_t<12, 12, false>(ut, W, nullptr, 12);                 // rows of ut are now U^T (V is not needed)
    epnp5_back(st, ut + 12 * 11, ut + 12 * 10, ut + 12 * 9, ut + 12 * 8, rvec, tvec, Rout);
}

// per-point DLT of cv::triangulatePoints: X4 = last row of V^T of the 4x4 system (stored float),
// then convertPointsFromHomogeneous in float, which divides by w only where |w| > FLT_EPSILON (strictly; a NaN w
// fails the test) and otherwise keeps scale 1: a zero-disparity point (w ~ 1e-18 from the DLT) comes out as the
// unit-norm column, not as a point 1e17 away.
// out4 (optional): the unit-norm homogeneous 4-vector itself, i.e. the column cv::triangulatePoints stores.
VO_HDN inline void triangulate_dlt(const double* Pl, const double* Pr, float xl, float yl, float xr, float yr,
                                   float* out3, float* out4 = nullptr)
{
    double At[16], W[4], Vt[16];
    const double x = xl, y = yl, x2 = xr, y2 = yr;
    for (int k = 0; k < 4; k++) {
        // A row-major rows: x*P[2]-P[0], y*P[2]-P[1] for both cameras; At = A^T
        At[k * 4 + 0] = x * Pl[8 + k] - Pl[k];
        At[k * 4 + 1] = y * Pl[8 + k] - Pl[4 + k];
        At[k * 4 + 2] = x2 * Pr[8 + k] - Pr[k];
        At[k * 4 + 3] = y2 * Pr[8 + k] - Pr[4 + k];
    }
    jacobi_svd_t<4, 4>(At, W, Vt, 4);
    const float X0 = (float)Vt[12], X1 = (float)Vt[13], X2 = (float)Vt[14], X3 = (float)Vt[15];
    if (out4) { out4[0] = X0; out4[1] = X1; out4[2] = X2; out4[3] = X3; }
    const float scale = fabsf(X3) > FLT_EPSILON ? 1.f / X3 : 1.f;
    out3[0] = X0 * scale; out3[1] = X1 * scale; out3[2] = X2 * scale;
}

} // namespace vomath
