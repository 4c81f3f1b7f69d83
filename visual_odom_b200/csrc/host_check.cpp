// host_check.cpp -- compiles the host/device math of pnp_math.cuh for the HOST so that the CPU test
// suite (-m "not gpu") can check the exact code the CUDA kernels run against cv2, without a GPU.
// It is a test hook of the product's own math, not a fallback: nothing in the library calls it.
#include "pnp_math.cuh"
#include "ess_math.cuh"
#include "p3p_math.cuh"
#include <vector>
extern "C" {
__attribute__((visibility("default"))) void vo_hostcheck_epnp5(const float* X, const float* uv, const float* K9, double* rvec, double* tvec, double* R)
{
    vomath::epnp5(X, uv, (double)K9[0], (double)K9[4], (double)K9[2], (double)K9[5], rvec, tvec, R);
}
__attribute__((visibility("default"))) void vo_hostcheck_triangulate(const float* Pl12, const float* Pr12, const float* a, const float* b, int n, float* X)
{
    double Pl[12], Pr[12];
    for (int k = 0; k < 12; k++) { Pl[k] = Pl12[k]; Pr[k] = Pr12[k]; }
    for (int i = 0; i < n; i++) vomath::triangulate_dlt(Pl, Pr, a[2 * i], a[2 * i + 1], b[2 * i], b[2 * i + 1], X + 3 * i);
}
// the same, with the unit-norm homogeneous column k_triangulate stores for vo_triangulate_homogeneous (n x 4)
__attribute__((visibility("default"))) void vo_hostcheck_triangulate4(const float* Pl12, const float* Pr12, const float* a, const float* b, int n, float* X, float* X4)
{
    double Pl[12], Pr[12];
    for (int k = 0; k < 12; k++) { Pl[k] = Pl12[k]; Pr[k] = Pr12[k]; }
    for (int i = 0; i < n; i++)
        vomath::triangulate_dlt(Pl, Pr, a[2 * i], a[2 * i + 1], b[2 * i], b[2 * i + 1], X + 3 * i, X4 + 4 * i);
}
__attribute__((visibility("default"))) void vo_hostcheck_rodrigues(const double* r, double* R, double* r_back)
{
    vomath::rodrigues_fwd(r, R);
    vomath::rodrigues_inv(R, r_back);
}
// the n == 4 case of solvePnPRansac as k_pnp_finalize runs it: returns 1 and (rvec, tvec, R = Rodrigues(rvec)) or 0
__attribute__((visibility("default"))) int vo_hostcheck_p3p(const float* X4, const float* uv4, const float* K9, double* rvec, double* tvec, double* R)
{
    double Rp[9];
    if (!vomath::p3p_four_points(X4, uv4, (double)K9[0], (double)K9[4], (double)K9[2], (double)K9[5], Rp, tvec)) return 0;
    vomath::rodrigues_inv(Rp, rvec);
    vomath::rodrigues_fwd(rvec, R);
    return 1;
}
// the LM step solve of k_pnp_finalize: returns 1 if it took the Cholesky path, 0 if OpenCV's SVD solve
__attribute__((visibility("default"))) int vo_hostcheck_lm_solve6(const double* JtJ, const double* JtErr, double lambda, double* dx)
{
    return vomath::lm_solve6(JtJ, JtErr, lambda, dx) ? 1 : 0;
}
__attribute__((visibility("default"))) int vo_hostcheck_five_point(const double* q1, const double* q2, double* E_out)
{
    return vomath::five_point(q1, q2, E_out);
}
// the whole mono branch on the host with the kernels' math: findEssentialMat(RANSAC, prob, thr) + recoverPose
__attribute__((visibility("default"))) int vo_hostcheck_mono_rotation(const float* p0, const float* p1, int n, double focal, double ppx, double ppy,
                                                                    double prob, double threshold, int max_iters, double* E_best, unsigned char* mask,
                                                                    double* R_out, int* iters_out)
{
    using namespace vomath;
    std::vector<double> q0(2 * n), q1(2 * n);
    for (int i = 0; i < n; i++) {
        q0[2 * i] = ((double)p0[2 * i] - ppx) / focal; q0[2 * i + 1] = ((double)p0[2 * i + 1] - ppy) / focal;
        q1[2 * i] = ((double)p1[2 * i] - ppx) / focal; q1[2 * i + 1] = ((double)p1[2 * i + 1] - ppy) / focal;
    }
    const double thr = threshold / focal;
    const float t = (float)(thr * thr);
    Rng rng(0xffffffffffffffffULL);
    int niters = max_iters, max_good = 0, it = 0;
    bool have = false;
    if (n == 5) {
        // no RANSAC: every candidate of one solve comes back stacked, recoverPose accepts only a single (3 x 3) one
        double Es[90];
        const int nm = five_point(q0.data(), q1.data(), Es);
        if (iters_out) *iters_out = 0;
        if (nm != 1) return 0;
        for (int k = 0; k < 9; k++) E_best[k] = Es[k];
        max_good = 5; have = true;
        niters = 0;
    }
    for (; it < niters; it++) {
        int idx[5];
        for (int i = 0; i < 5; i++) {
            int v; bool dup;
            do { v = (int)(rng.next() % (unsigned)n); dup = false; for (int j = 0; j < i; j++) dup |= idx[j] == v; } while (dup);
            idx[i] = v;
        }
        double a[10], b[10], Es[90];
        for (int i = 0; i < 5; i++) { a[2 * i] = q0[2 * idx[i]]; a[2 * i + 1] = q0[2 * idx[i] + 1]; b[2 * i] = q1[2 * idx[i]]; b[2 * i + 1] = q1[2 * idx[i] + 1]; }
        const int nm = five_point(a, b, Es);
        for (int m = 0; m < nm; m++) {
            int good = 0;
            for (int i = 0; i < n; i++) good += sampson_err(Es + 9 * m, q0[2 * i], q0[2 * i + 1], q1[2 * i], q1[2 * i + 1]) <= t;
            if (good > (max_good > 4 ? max_good : 4)) {
                max_good = good; have = true;
                for (int k = 0; k < 9; k++) E_best[k] = Es[9 * m + k];
                niters = ransac_update_num_iters(prob, (double)(n - good) / n, 5, niters);
            }
        }
    }
    if (iters_out) *iters_out = it;
    if (!have) return 0;
    for (int i = 0; i < n; i++) mask[i] = n == 5 || sampson_err(E_best, q0[2 * i], q0[2 * i + 1], q1[2 * i], q1[2 * i + 1]) <= t;
    double R1[9], R2[9], tt[3], tn[3];
    decompose_essential(E_best, R1, R2, tt);
    for (int k = 0; k < 3; k++) tn[k] = -tt[k];
    const double* Rs[4] = {R1, R2, R1, R2};
    const double* ts[4] = {tt, tt, tn, tn};
    int good[4] = {0, 0, 0, 0};
    for (int c = 0; c < 4; c++)
        for (int i = 0; i < n; i++)
            if (mask[i] && cheirality_ok(Rs[c], ts[c], q0[2 * i], q0[2 * i + 1], q1[2 * i], q1[2 * i + 1], 50.0)) good[c]++;
    int k = 3;
    if (good[0] >= good[1] && good[0] >= good[2] && good[0] >= good[3]) k = 0;
    else if (good[1] >= good[0] && good[1] >= good[2] && good[1] >= good[3]) k = 1;
    else if (good[2] >= good[0] && good[2] >= good[1] && good[2] >= good[3]) k = 2;
    for (int j = 0; j < 9; j++) R_out[j] = Rs[k][j];
    return max_good;
}
}
