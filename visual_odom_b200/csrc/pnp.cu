// pnp.cu -- K5 triangulation + K6 PnP/RANSAC (hypotheses, batched reprojection residuals,
// sequential replay of OpenCV's best-model / adaptive-iteration rule, Levenberg-Marquardt refine).
//
// Replaces
//   cv::triangulatePoints + cv::convertPointsFromHomogeneous        reference src/main.cpp:170-171
//   cv::solvePnPRansac(X, x, K, 0, rvec=0, t_prev, true, 500, 0.5, 0.999, inliers, SOLVEPNP_ITERATIVE)
//   + cv::Rodrigues                                                  reference src/visualOdometry.cpp:161-189
// Restated in oracle/pnp_ref.py (pinned against cv2: EPnP models bit-exact, inlier masks identical).
//
// Structure (all per work unit, no host round trip):
//   k_triangulate        one thread per point: 4x4 DLT via Jacobi SVD in fp64, f32 out
//   waves of RANSAC iterations [0,32) [32,128) [128,iters): a unit that has already reached its
//   adaptive iteration count skips the remaining waves
//     k_pnp_subsets      1 thread/unit: cv::RNG(2^64-1) stream -> 5 distinct indices per iteration
//     k_pnp_hypotheses   1 thread/iteration: 5-point EPnP in fp64 (pnp_math.cuh) -> [R|t]
//     k_pnp_count        1 CTA/iteration: project all N points (fp64 -> f32), err^2 <= 0.25f, count
//     k_pnp_replay       1 thread/unit: `if count > max(best,4)`: new best, niters = RANSACUpdateNumIters
//   k_pnp_init           per unit: RNG / bound reset; n == 5 (no RANSAC in OpenCV): the single unrefined EPnP
//   k_pnp_finalize       1 CTA/unit (n == 4: OpenCV's P3P case, no RANSAC): inlier mask of the best model -> ordered index list; LM
//                        (CvLevMarq logic, lambda 1e-3, <=20 iterations, eps FLT_EPSILON) over the
//                        inliers from (rvec=0, t_prev); Rodrigues.
#include "common.cuh"
#include "pnp.h"
#include "pnp_math.cuh"
#include "p3p_math.cuh"

using namespace vomath;

__global__ void k_triangulate(const TriArgs a)
{
    const int unit = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = a.n_pts[unit];
    if (i >= n) return;
    const float2 pl = a.pts_l[(size_t)unit * a.cap + i];
    const float2 pr = a.pts_r[(size_t)unit * a.cap + i];
    float o[3], o4[4];
    const CamCalib& c = a.cal[unit];
    triangulate_dlt(c.Pl, c.Pr, pl.x, pl.y, pr.x, pr.y, o, o4);
    a.X[(size_t)unit * a.cap + i] = make_float3(o[0], o[1], o[2]);
    if (a.X4) a.X4[(size_t)unit * a.cap + i] = make_float4(o4[0], o4[1], o4[2], o4[3]);
}

// ---------------------------------------------------------------------------------------------
// Exactly five correspondences (= model points): OpenCV runs no RANSAC, one EPnP solvePnP on all five, no refinement,
// all five inliers.  It reports success whatever EPnP returns: five identical points give rvec = 0 and a nan tvec, and
// so does this.  Kept out of line and out of k_pnp_finalize, whose LM would spill around the 12x12 SVD.
__device__ __noinline__ void pnp_five_points(const PnpArgs& a, int unit)
{
    const float3* X = a.X + (size_t)unit * a.cap;
    const float2* x = a.x + (size_t)unit * a.cap;
    float Xw[15], uv[10];
    for (int i = 0; i < 5; i++) {
        Xw[3 * i] = X[i].x; Xw[3 * i + 1] = X[i].y; Xw[3 * i + 2] = X[i].z;
        uv[2 * i] = x[i].x; uv[2 * i + 1] = x[i].y;
    }
    double rv[3], t[3], R[9];
    const CamCalib& c = a.cal[unit];
    epnp5(Xw, uv, c.fu, c.fv, c.uc, c.vc, rv, t, R);      // R = Rodrigues(rvec), the caller's conversion
    vo_unit_result_dev& res = a.results[unit];
    int* inl = a.inliers + (size_t)unit * a.cap;
    res.ransac_iters = 0;
    res.n_inliers = 5;
    res.pnp_status = VO_PNP_OK;
    for (int i = 0; i < 5; i++) inl[i] = i;
    for (int k = 0; k < 3; k++) { res.rvec[k] = rv[k]; res.tvec[k] = t[k]; }
    for (int k = 0; k < 9; k++) res.R[k] = R[k];
}

__global__ void k_pnp_init(const PnpArgs a)
{
    const int unit = blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= a.n_units) return;
    PnpState& s = a.state[unit];
    s.rng_state = 0xffffffffffffffffULL;
    s.niters = a.par[unit].pnp_iterations;        // the unit's own bound (a.iterations is the scratch stride)
    s.max_good = 0;
    s.best_it = -1;
    s.iters_run = 0;
    const int n = a.n_pts[unit];
    // n < 4: the reference aborts; n == 4: no RANSAC, k_pnp_finalize runs the P3P solve; n == 5: no RANSAC, the EPnP solve
    s.done = (n <= 5) ? 1 : 0;
    if (n == 5) pnp_five_points(a, unit);
}

__global__ void k_pnp_subsets(const PnpArgs a, int it0, int it1)
{
    const int unit = blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= a.n_units) return;
    PnpState& s = a.state[unit];
    if (s.done) return;
    const int n = a.n_pts[unit];
    int* out = a.subsets + ((size_t)unit * a.iterations) * 5;
    Rng rng(s.rng_state);
    const int last = it1 < s.niters ? it1 : s.niters;
    for (int it = it0; it < last; it++) {
        int idx[5];                     // n > 5 here: smaller units are done before the first wave
        for (int i = 0; i < 5; i++) {
            int v;
            bool dup;
            do {
                v = (int)(rng.next() % (unsigned)n);
                dup = false;
                for (int j = 0; j < i; j++) dup |= (idx[j] == v);
            } while (dup);
            idx[i] = v;
        }
        for (int i = 0; i < 5; i++) out[it * 5 + i] = idx[i];
    }
    s.rng_state = rng.state;
}

// ---------------------------------------------------------------------------------------------
// Warp-cooperative one-sided Jacobi SVD of the symmetric 12x12 Gram matrix (U^T and W only).
// Lane r (< 12) of a 16-lane group owns row r of At in registers.  OpenCV sweeps the pairs (i, j) in
// row-major order; a pair only depends on earlier pairs that touch row i or row j, and all of those
// have a smaller i + j, so the pairs of one anti-diagonal (i + j = t) are independent: the sweep is
// run as 21 wavefronts of up to 6 disjoint pairs, each pair on its two row-owner lanes, with exactly
// the operations (and operation order) of jacobi_svd_t -- the result is bit-identical, 3x shorter.
// Returns false when a singular value is exactly zero (the caller then uses the sequential routine,
// which implements OpenCV's random-vector completion for that case).
__device__ bool jacobi12_coop(double (&row)[12], double& wout, int r, int gbase, unsigned gmask)
{
    const double eps = kDblEps * 10;
    const bool live = r < 12;
    double W = 0;
    for (int k = 0; k < 12; k++) W += row[k] * row[k];
    for (int iter = 0; iter < 30; iter++) {
        bool changed = false;
        for (int t = 1; t <= 21; t++) {
            const int partner = t - r;
            const bool active = live && partner >= 0 && partner < 12 && partner != r;
            const int src = gbase + (active ? partner : r);
            double other[12];
#pragma unroll
            for (int k = 0; k < 12; k++) other[k] = __shfl_sync(gmask, row[k], src);
            const double Wo = __shfl_sync(gmask, W, src);
            if (active) {
                const bool is_i = r < partner;
                const double a0 = is_i ? W : Wo, b0 = is_i ? Wo : W;
                double p = 0;
#pragma unroll
                for (int k = 0; k < 12; k++) p += row[k] * other[k];          // Ai[k]*Aj[k]: the product commutes
                if (!(fabs(p) <= eps * sqrt(a0 * b0))) {
                    p *= 2;
                    const double beta = a0 - b0, gamma = cv_hypot(p, beta);
                    double c, s;
                    if (beta < 0) {
                        const double delta = (gamma - beta) * 0.5;
                        s = sqrt(delta / gamma);
                        c = p / (gamma * s * 2);
                    } else {
                        c = sqrt((gamma + beta) / (gamma * 2));
                        s = p / (gamma * c * 2);
                    }
                    double acc = 0;
                    if (is_i) {
#pragma unroll
                        for (int k = 0; k < 12; k++) { const double t0 = c * row[k] + s * other[k]; row[k] = t0; acc += t0 * t0; }
                    } else {
#pragma unroll
                        for (int k = 0; k < 12; k++) { const double t1 = -s * other[k] + c * row[k]; row[k] = t1; acc += t1 * t1; }
                    }
                    W = acc;
                    changed = true;
                }
            }
        }
        if (!__any_sync(gmask, changed)) break;
    }
    double sd = 0;
    for (int k = 0; k < 12; k++) sd += row[k] * row[k];
    W = sqrt(sd);
    wout = W;
    return !__any_sync(gmask, live && W <= kDblMin);
}

// One iteration (hypothesis) per 16-lane group: the leader lane runs the scalar stages of EPnP
// (pnp_math.cuh), the 12 row-owner lanes run the SVD of the Gram matrix.
#define HYP_PER_CTA 2
__global__ void __launch_bounds__(32 * 1) k_pnp_hypotheses(const PnpArgs a, int it0, int it1)
{
    const int unit = blockIdx.y;
    const int lane = threadIdx.x & 31, g = lane >> 4, r = lane & 15;
    const int it = it0 + blockIdx.x * HYP_PER_CTA + g;
    const PnpState& s = a.state[unit];
    const bool work = !(s.done || it >= it1 || it >= s.niters);
    const unsigned gmask = 0xffffu << (16 * g);
    if (!__any_sync(0xffffffffu, work)) return;
    __shared__ double sm_mtm[HYP_PER_CTA][144];
    __shared__ double sm_ut[HYP_PER_CTA][48];        // rows 11, 10, 9, 8 of U^T
    __shared__ int sm_rank_ok[HYP_PER_CTA];
    __shared__ Epnp5State sm_st[HYP_PER_CTA];
    if (work && r == 0) {
        const int* idx = a.subsets + ((size_t)unit * a.iterations + it) * 5;
        float Xs[15], xs[10];
        for (int i = 0; i < 5; i++) {
            const float3 P = a.X[(size_t)unit * a.cap + idx[i]];
            const float2 p = a.x[(size_t)unit * a.cap + idx[i]];
            Xs[3 * i] = P.x; Xs[3 * i + 1] = P.y; Xs[3 * i + 2] = P.z;
            xs[2 * i] = p.x; xs[2 * i + 1] = p.y;
        }
        const CamCalib& c = a.cal[unit];
        epnp5_front(Xs, xs, c.fu, c.fv, c.uc, c.vc, sm_st[g], sm_mtm[g]);
    }
    __syncwarp();
    if (work) {          // uniform per 16-lane group
        double row[12], W;
#pragma unroll
        for (int k = 0; k < 12; k++) row[k] = (r < 12) ? sm_mtm[g][r * 12 + k] : 0.0;
        const bool ok = jacobi12_coop(row, W, r, 16 * g, gmask);
        // OpenCV then orders the rows by descending W with a selection sort (first maximum wins, swap);
        // every lane replays it on the 12 values to learn which original row lands at positions 8..11
        double Wv[12];
        int id[12];
#pragma unroll
        for (int k = 0; k < 12; k++) { Wv[k] = __shfl_sync(gmask, W, 16 * g + k); id[k] = k; }
#pragma unroll
        for (int i = 0; i < 11; i++) {
            int best = i, bid = id[i];
            double bv = Wv[i];
#pragma unroll
            for (int k = i + 1; k < 12; k++)
                if (bv < Wv[k]) { bv = Wv[k]; best = k; bid = id[k]; }
            const double wi = Wv[i];
            const int ii = id[i];
#pragma unroll
            for (int k = i + 1; k < 12; k++)
                if (k == best) { Wv[k] = wi; id[k] = ii; }
            Wv[i] = bv; id[i] = bid;
        }
        if (r < 12) {
            const double sc = W > kDblMin ? 1 / W : 0.;
#pragma unroll
            for (int q = 0; q < 4; q++)
                if (id[11 - q] == r) {
#pragma unroll
                    for (int k = 0; k < 12; k++) sm_ut[g][q * 12 + k] = row[k] * sc;
                }
        }
        if (r == 0) sm_rank_ok[g] = ok ? 1 : 0;
    }
    __syncwarp();
    // EPnP tail: the three beta approximations are independent -> lanes 0..2 of the group run one each in lockstep
    // (same instruction stream, run-time system width), lane 0 then picks like the reference (N = 1; 2 if err2 < err1;
    // 3 if err3 < the best so far).  A rank-deficient M^T M (exactly-zero singular value) takes the sequential routine.
    const bool fast_tail = work && sm_rank_ok[g];
    double Rk[9], tk[3], errk = 0;
    if (fast_tail && r < 3)
        epnp5_back_one(sm_st[g], sm_ut[g], sm_ut[g] + 12, sm_ut[g] + 24, sm_ut[g] + 36, r + 1, Rk, tk, &errk);
    __syncwarp();
    if (fast_tail) {          // uniform per 16-lane group
        const double e1 = __shfl_sync(gmask, errk, 16 * g + 1), e2 = __shfl_sync(gmask, errk, 16 * g + 2);
        int pick = 0;
        double best = errk;                       // lane 0's own value is approximation 1
        if (r == 0) {
            if (e1 < best) { best = e1; pick = 1; }
            if (e2 < best) { best = e2; pick = 2; }
        }
        pick = __shfl_sync(gmask, pick, 16 * g);
#pragma unroll
        for (int k = 0; k < 9; k++) Rk[k] = __shfl_sync(gmask, Rk[k], 16 * g + pick);
#pragma unroll
        for (int k = 0; k < 3; k++) tk[k] = __shfl_sync(gmask, tk[k], 16 * g + pick);
    }
    if (work && r == 0) {
        double rvec[3], tvec[3], R[9];
        if (fast_tail) {
            rodrigues_inv(Rk, rvec);
            for (int k = 0; k < 3; k++) tvec[k] = tk[k];
            rodrigues_fwd(rvec, R);               // computeError -> projectPoints(rvec) converts back with Rodrigues
        } else {        // exactly-zero singular value: the sequential routine handles OpenCV's completion rule
            double ut[144], W12[12];
            for (int k = 0; k < 144; k++) ut[k] = sm_mtm[g][k];
            jacobi_svd_t<12, 12, false>(ut, W12, nullptr, 12);
            epnp5_back(sm_st[g], ut + 12 * 11, ut + 12 * 10, ut + 12 * 9, ut + 12 * 8, rvec, tvec, R);
        }
        double* m = a.models + ((size_t)unit * a.iterations + it) * 12;
        for (int k = 0; k < 9; k++) m[k] = R[k];
        for (int k = 0; k < 3; k++) m[9 + k] = tvec[k];
    }
}

__device__ __forceinline__ float reproj_err(const double* m, float3 P, float2 p, double fu, double fv, double uc, double vc)
{
    const double X = P.x, Y = P.y, Z = P.z;
    double x = m[0] * X + m[1] * Y + m[2] * Z + m[9];
    double y = m[3] * X + m[4] * Y + m[5] * Z + m[10];
    double z = m[6] * X + m[7] * Y + m[8] * Z + m[11];
    z = z ? 1. / z : 1.;
    x *= z; y *= z;
    const float u = (float)(x * fu + uc), v = (float)(y * fv + vc);
    const float dx = p.x - u, dy = p.y - v;
    return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}

__global__ void __launch_bounds__(128) k_pnp_count(const PnpArgs a, int it0, int it1)
{
    const int unit = blockIdx.y;
    const int it = it0 + blockIdx.x;
    const PnpState& s = a.state[unit];
    if (s.done || it >= it1 || it >= s.niters) return;
    __shared__ double m[12], cam[4];         // the model; the unit's fu, fv, uc, vc
    __shared__ int total;
    const float thr2 = a.par[unit].thr2;
    if (threadIdx.x < 12) m[threadIdx.x] = a.models[((size_t)unit * a.iterations + it) * 12 + threadIdx.x];
    else if (threadIdx.x < 16) cam[threadIdx.x - 12] = (&a.cal[unit].fu)[threadIdx.x - 12];
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    const int n = a.n_pts[unit];
    int c = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float e = reproj_err(m, a.X[(size_t)unit * a.cap + i], a.x[(size_t)unit * a.cap + i], cam[0], cam[1], cam[2], cam[3]);
        c += (e <= thr2) ? 1 : 0;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31) == 0) atomicAdd(&total, c);
    __syncthreads();
    if (threadIdx.x == 0) a.counts[(size_t)unit * a.iterations + it] = total;
}

__global__ void k_pnp_replay(const PnpArgs a, int it0, int it1)
{
    const int unit = blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= a.n_units) return;
    PnpState& s = a.state[unit];
    if (s.done) return;
    const int n = a.n_pts[unit];
    const int* cnt = a.counts + (size_t)unit * a.iterations;
    int it = it0;
    for (; it < it1 && it < s.niters; it++) {
        const int good = cnt[it];
        if (good > max(s.max_good, 4)) {
            s.best_it = it;
            s.max_good = good;
            s.niters = ransac_update_num_iters(a.par[unit].confidence, (double)(n - good) / n, 5, s.niters);
        }
    }
    s.iters_run = it;
    if (it >= s.niters || it1 >= a.par[unit].pnp_iterations) s.done = 1;
}

// ---------------------------------------------------------------------------------------------
// Block-wide sum of NV doubles per thread -> result broadcast in smem red[0..NV)
template <int NV>
__device__ void block_reduce(double (&v)[NV], double* red /* [NV] */, double* scratch /* [warps*NV] */)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; k++) {
        double x = v[k];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d);
        if (lane == 0) scratch[warp * NV + k] = x;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        double x = 0;
        for (int w = 0; w < nw; w++) x += scratch[w * NV + threadIdx.x];
        red[threadIdx.x] = x;
    }
    __syncthreads();
}

// dR/dr_j (OpenCV's Rodrigues jacobian layout), used by the LM jacobian
__device__ void rodrigues_jac(const double* r, double* J /* 3 x 9 */)
{
    const double theta = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    for (int k = 0; k < 27; k++) J[k] = 0;
    if (theta < kDblEps) {
        J[5] = -1; J[7] = 1; J[9 + 2] = 1; J[9 + 6] = -1; J[18 + 1] = -1; J[18 + 3] = 1;
        return;
    }
    const double c = cos(theta), s = sin(theta), c1 = 1. - c, itheta = 1. / theta;
    const double k[3] = {r[0] * itheta, r[1] * itheta, r[2] * itheta};
    const double rrt[9] = {k[0] * k[0], k[0] * k[1], k[0] * k[2], k[0] * k[1], k[1] * k[1], k[1] * k[2], k[0] * k[2], k[1] * k[2], k[2] * k[2]};
    const double r_x[9] = {0, -k[2], k[1], k[2], 0, -k[0], -k[1], k[0], 0};
    const double drrt[27] = {2 * k[0], k[1], k[2], k[1], 0, 0, k[2], 0, 0,
                             0, k[0], 0, k[0], 2 * k[1], k[2], 0, k[2], 0,
                             0, 0, k[0], 0, 0, k[1], k[0], k[1], 2 * k[2]};
    const double d_r_x[27] = {0, 0, 0, 0, 0, -1, 0, 1, 0,
                              0, 0, 1, 0, 0, 0, -1, 0, 0,
                              0, -1, 0, 1, 0, 0, 0, 0, 0};
    for (int i = 0; i < 3; i++) {
        const double ri = k[i];
        const double a0 = -s * ri, a1 = (s - 2 * c1 * itheta) * ri, a2 = c1 * itheta, a3 = (c - s * itheta) * ri, a4 = s * itheta;
        for (int q = 0; q < 9; q++)
            J[i * 9 + q] = a0 * ((q % 4 == 0) ? 1. : 0.) + a1 * rrt[q] + a2 * drrt[i * 9 + q] + a3 * r_x[q] + a4 * d_r_x[i * 9 + q];
    }
}

#define FIN_T 256
// one CTA per unit: minBlocks = 1 lets ptxas use up to 255 registers (with FIN_T alone it stopped at 128 and spilled the
// LM accumulators)
__global__ void __launch_bounds__(FIN_T, 1) k_pnp_finalize(const PnpArgs a)
{
    const int unit = blockIdx.x;
    const PnpState& st = a.state[unit];
    const int n = a.n_pts[unit];
    vo_unit_result_dev& res = a.results[unit];
    const float3* X = a.X + (size_t)unit * a.cap;
    const float2* x = a.x + (size_t)unit * a.cap;
    int* inl = a.inliers + (size_t)unit * a.cap;

    __shared__ double sm_model[12], cam[4];      // the best model; the unit's fu, fv, uc, vc
    __shared__ int wcnt[FIN_T / 32];
    __shared__ int base;
    __shared__ double red[28];
    __shared__ double scratch[(FIN_T / 32) * 28];
    __shared__ double param[6], prev_param[6], JtJ[36], JtErr[6];
    __shared__ int ctrl;          // loop control broadcast
    __shared__ double shared_norm;

    const double* t_prev = a.t_prev + 3 * unit;
    if (n == 4) {
        // exactly four correspondences: OpenCV runs no RANSAC, one P3P solvePnP on all four, no refinement, all four inliers
        if (threadIdx.x == 0) {
            float Xw[12], uv[8];
            for (int i = 0; i < 4; i++) {
                Xw[3 * i] = X[i].x; Xw[3 * i + 1] = X[i].y; Xw[3 * i + 2] = X[i].z;
                uv[2 * i] = x[i].x; uv[2 * i + 1] = x[i].y;
            }
            double R[9], t[3], rv[3];
            const CamCalib& c = a.cal[unit];
            const bool ok = p3p_four_points(Xw, uv, c.fu, c.fv, c.uc, c.vc, R, t);
            res.ransac_iters = 0;
            if (ok) {
                rodrigues_inv(R, rv);
                rodrigues_fwd(rv, R);                  // the caller's cv::Rodrigues(rvec, rotation), visualOdometry.cpp:180
                res.n_inliers = 4;
                res.pnp_status = VO_PNP_OK;
                for (int i = 0; i < 4; i++) inl[i] = i;
                for (int k = 0; k < 3; k++) { res.rvec[k] = rv[k]; res.tvec[k] = t[k]; }
                for (int k = 0; k < 9; k++) res.R[k] = R[k];
            } else {
                res.n_inliers = 0;
                res.pnp_status = VO_PNP_NO_MODEL;
                for (int k = 0; k < 3; k++) { res.rvec[k] = 0; res.tvec[k] = t_prev[k]; }
                for (int k = 0; k < 9; k++) res.R[k] = (k % 4 == 0) ? 1. : 0.;
            }
        }
        return;
    }
    if (n == 5) return;             // k_pnp_init wrote the record (pnp_five_points)
    if (st.best_it < 0 || n < 4) {
        // solvePnPRansac returns false: rvec / tvec stay what the caller passed in
        if (threadIdx.x == 0) {
            res.n_inliers = 0;
            res.ransac_iters = st.iters_run;
            res.pnp_status = (n < 4) ? VO_PNP_TOO_FEW : VO_PNP_NO_MODEL;
            for (int k = 0; k < 3; k++) { res.rvec[k] = 0; res.tvec[k] = t_prev[k]; }
            for (int k = 0; k < 9; k++) res.R[k] = (k % 4 == 0) ? 1. : 0.;
        }
        return;
    }
    if (threadIdx.x < 12) sm_model[threadIdx.x] = a.models[((size_t)unit * a.iterations + st.best_it) * 12 + threadIdx.x];
    else if (threadIdx.x < 16) cam[threadIdx.x - 12] = (&a.cal[unit].fu)[threadIdx.x - 12];
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    const double fu = cam[0], fv = cam[1], uc = cam[2], vc = cam[3];
    const float thr2 = a.par[unit].thr2;
    // ---- inlier mask of the best model, ordered compaction -----------------------------------
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c0 = 0; c0 < n; c0 += FIN_T) {
        const int i = c0 + threadIdx.x;
        bool keep = false;
        if (i < n) keep = reproj_err(sm_model, X[i], x[i], fu, fv, uc, vc) <= thr2;
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) wcnt[warp] = __popc(b);
        __syncthreads();
        int off = base;
        for (int w = 0; w < warp; w++) off += wcnt[w];
        if (keep) inl[off + __popc(b & ((1u << lane) - 1u))] = i;
        __syncthreads();
        if (threadIdx.x == 0) {
            int t = 0;
            for (int w = 0; w < FIN_T / 32; w++) t += wcnt[w];
            base += t;
        }
        __syncthreads();
    }
    const int nin = base;

    // ---- Levenberg-Marquardt over the inliers (CvLevMarq state machine) ----------------------
    if (threadIdx.x < 3) { param[threadIdx.x] = 0.; param[3 + threadIdx.x] = t_prev[threadIdx.x]; }
    __syncthreads();
    int lambda_lg10 = -3, iters = 0;
    double prev_err_norm = 0;
    // evaluates residuals (and optionally J^T J, J^T e) at `param`; result norm in shared_norm
    auto evaluate = [&](bool with_jac) {
        double R[9], dRdr[27];
        rodrigues_fwd(param, R);
        if (with_jac) rodrigues_jac(param, dRdr);
        double acc[28];
#pragma unroll
        for (int k = 0; k < 28; k++) acc[k] = 0;
        for (int q = threadIdx.x; q < nin; q += FIN_T) {
            const float3 P = X[inl[q]];
            const float2 p = x[inl[q]];
            const double Xw = P.x, Yw = P.y, Zw = P.z;
            const double xc = R[0] * Xw + R[1] * Yw + R[2] * Zw + param[3];
            const double yc = R[3] * Xw + R[4] * Yw + R[5] * Zw + param[4];
            double zc = R[6] * Xw + R[7] * Yw + R[8] * Zw + param[5];
            const double z = zc ? 1. / zc : 1.;
            const double xn = xc * z, yn = yc * z;
            const double ex = xn * fu + uc - (double)p.x, ey = yn * fv + vc - (double)p.y;
            acc[27] += ex * ex + ey * ey;
            if (with_jac) {
                double jx[6], jy[6];
                for (int j = 0; j < 3; j++) {
                    const double* dR = dRdr + 9 * j;
                    const double dx = dR[0] * Xw + dR[1] * Yw + dR[2] * Zw;
                    const double dy = dR[3] * Xw + dR[4] * Yw + dR[5] * Zw;
                    const double dz = dR[6] * Xw + dR[7] * Yw + dR[8] * Zw;
                    jx[j] = fu * z * (dx - xn * dz);
                    jy[j] = fv * z * (dy - yn * dz);
                }
                jx[3] = fu * z; jx[4] = 0; jx[5] = -fu * xn * z;
                jy[3] = 0; jy[4] = fv * z; jy[5] = -fv * yn * z;
                int q2 = 0;
                for (int r = 0; r < 6; r++)
                    for (int c = r; c < 6; c++) acc[q2++] += jx[r] * jx[c] + jy[r] * jy[c];
                for (int r = 0; r < 6; r++) acc[21 + r] += jx[r] * ex + jy[r] * ey;
            }
        }
        block_reduce<28>(acc, red, scratch);
        if (threadIdx.x == 0) {
            shared_norm = sqrt(red[27]);
            if (with_jac) {
                int q2 = 0;
                for (int r = 0; r < 6; r++)
                    for (int c = r; c < 6; c++) { JtJ[r * 6 + c] = red[q2]; JtJ[c * 6 + r] = red[q2]; q2++; }
                for (int r = 0; r < 6; r++) JtErr[r] = red[21 + r];
            }
        }
        __syncthreads();
    };
    auto lm_step = [&]() {      // thread 0: param = prev_param - solve((JtJ with scaled diagonal), JtErr)
        if (threadIdx.x == 0) {
            const double lambda = exp(lambda_lg10 * log(10.));
            // (J^T J + lambda diag) dx = J^T e: Cholesky while positive definite, OpenCV's SVD solve otherwise
            // (lm_solve6 in pnp_math.cuh; the refined pose is pinned to cv2 at 1e-8 by tests/test_gpu_pnp_refine.py)
            double dx[6];
            lm_solve6(JtJ, JtErr, lambda, dx);
            for (int k = 0; k < 6; k++) param[k] = prev_param[k] - dx[k];
        }
        __syncthreads();
    };
    evaluate(true);
    for (;;) {
        if (threadIdx.x < 6) prev_param[threadIdx.x] = param[threadIdx.x];
        __syncthreads();
        if (iters == 0) prev_err_norm = shared_norm;
        lm_step();
        double err_norm;
        for (;;) {
            evaluate(false);
            err_norm = shared_norm;
            if (err_norm > prev_err_norm) {
                if (++lambda_lg10 <= 16) { lm_step(); continue; }
            }
            break;
        }
        lambda_lg10 = max(lambda_lg10 - 1, -16);
        if (threadIdx.x == 0) {
            double dn = 0, pn = 0;
            for (int k = 0; k < 6; k++) { const double d = param[k] - prev_param[k]; dn += d * d; pn += prev_param[k] * prev_param[k]; }
            ctrl = (++iters >= 20 || sqrt(dn) / (sqrt(pn) + kDblEps) < 1.1920928955078125e-07) ? 1 : 0;
        } else {
            ++iters;
        }
        __syncthreads();
        if (ctrl) break;
        prev_err_norm = err_norm;
        evaluate(true);
    }
    if (threadIdx.x == 0) {
        res.n_inliers = nin;
        res.ransac_iters = st.iters_run;
        res.pnp_status = VO_PNP_OK;
        for (int k = 0; k < 3; k++) { res.rvec[k] = param[k]; res.tvec[k] = param[3 + k]; }
        double R[9];
        rodrigues_fwd(param, R);
        for (int k = 0; k < 9; k++) res.R[k] = R[k];
    }
}

// ---------------------------------------------------------------------------------------------
int vo_launch_triangulate(const TriArgs& a, int n_units, cudaStream_t stream)
{
    dim3 g((a.cap + 127) / 128, n_units);
    k_triangulate<<<g, 128, 0, stream>>>(a);
    return 1;
}

int vo_launch_pnp(const PnpArgs& a, cudaStream_t stream)
{
    int launches = 0;
    const int ub = (a.n_units + 63) / 64;
    k_pnp_init<<<ub, 64, 0, stream>>>(a);
    launches++;
    const int waves[4] = {0, 32, 128, a.iterations};
    for (int w = 0; w < 3; w++) {
        int it0 = waves[w], it1 = waves[w + 1];
        if (it1 > a.iterations) it1 = a.iterations;
        if (it0 >= it1) continue;
        k_pnp_subsets<<<ub, 64, 0, stream>>>(a, it0, it1);
        dim3 gh((it1 - it0 + 1) / 2, a.n_units);          // two hypotheses (16-lane groups) per warp
        k_pnp_hypotheses<<<gh, 32, 0, stream>>>(a, it0, it1);
        dim3 gc(it1 - it0, a.n_units);
        k_pnp_count<<<gc, 128, 0, stream>>>(a, it0, it1);
        k_pnp_replay<<<ub, 64, 0, stream>>>(a, it0, it1);
        launches += 4;
    }
    k_pnp_finalize<<<a.n_units, FIN_T, 0, stream>>>(a);
    launches++;
    return launches;
}
