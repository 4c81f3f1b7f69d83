// ess.cu -- the `mono_rotation = true` branch of the reference's trackingFrame2Frame
// (reference src/visualOdometry.cpp:146-157):
//     E = cv::findEssentialMat(pointsLeft_t0, pointsLeft_t1, focal, pp, cv::RANSAC, 0.999, 1.0, mask);
//     cv::recoverPose(E, pointsLeft_t0, pointsLeft_t1, rotation, translation_mono, focal, pp, mask);
// The reference's main() passes mono_rotation = false (src/main.cpp:181), but the flag's header default is true
// (src/visualOdometry.h:42), so a drop-in must honour it.
//
// Structure (same shape as the PnP RANSAC of pnp.cu: waves of iterations, a unit that reached its adaptive bound skips
// the rest; every kernel reads the point count and the bound from device memory, so there is no host round trip and the
// launch sequence is the same for every count -- the sequence mode captures it in the frame's graph):
//   k_ess_init          normalise the points ((p - pp) / focal in fp64), reset the RANSAC state
//   k_ess_five          n == 5 only, instead of the RANSAC waves: one five-point solve on all points (no RANSAC in OpenCV);
//                       n < 5 runs neither (no model: the reference aborts)
//   k_ess_subsets       1 thread / problem: cv::RNG(2^64-1) stream -> 5 distinct indices per iteration (ptsetreg.cpp getSubset)
//   k_ess_hypotheses    1 thread / iteration: Nister five-point solver (ess_math.cuh) -> up to 10 E per sample
//   k_ess_count         1 CTA / (iteration, candidate): Sampson error of all N points, err <= (float)thr^2, count
//   k_ess_replay        1 thread / problem: candidates in order, `count > max(best, 4)` -> new best, RANSACUpdateNumIters
//   k_ess_mask          inlier mask of the best E
//   k_ess_decompose     1 thread / problem: decomposeEssentialMat
//   k_ess_cheirality    1 thread / point: the four [R|t] hypotheses of recoverPose (fp64 DLT, distance threshold 50)
//   k_ess_pick          1 thread / problem: recoverPose's vote -> rotation
// One launch serves n_prob independent problems (EssArgs strides): the grid kernels take theirs from blockIdx.y
// (k_ess_count, whose x and y are (iteration, candidate), from blockIdx.z), the per-problem bookkeeping kernels run one
// thread per problem.  Only the addressing depends on the problem count, so each problem's results are bit for bit those
// of running it alone, and a problem that reached its adaptive bound skips the later waves while the others go on.
// Restated in oracle/essential_ref.py; the math of ess_math.cuh is checked on the host against cv2 4.13.0
// (tests/test_oracle_essential.py) and on the GPU through vo_mono_rotation (tests/test_gpu_stages.py).
#include "common.cuh"
#include "ess.h"
#include "ess_math.cuh"

using namespace vomath;

// the point count of this run; n_max sizes every per-point buffer, so a count beyond it is clamped rather than overrun
static __device__ __forceinline__ int ess_n(const EssArgs& a)
{
    const int n = *a.n;
    return n < 0 ? 0 : (n < a.n_max ? n : a.n_max);
}

template <typename T> static __device__ __forceinline__ T* ess_at(T* ptr, size_t bytes)
{
    return (T*)((const char*)ptr + bytes);
}

// problem p's arguments: every pointer moved by its stride
static __device__ __forceinline__ EssArgs ess_prob(const EssArgs& a0, int p)
{
    EssArgs a = a0;
    const size_t so = (size_t)p * a0.scratch_stride;
    a.n += (size_t)p * a0.n_stride;
    a.cal += (size_t)p * a0.cal_stride;
    a.pts0 += (size_t)p * a0.pts_stride; a.pts1 += (size_t)p * a0.pts_stride;
    a.q0 = ess_at(a0.q0, so); a.q1 = ess_at(a0.q1, so); a.state = ess_at(a0.state, so);
    a.subsets = ess_at(a0.subsets, so); a.models = ess_at(a0.models, so); a.nmodels = ess_at(a0.nmodels, so);
    a.counts = ess_at(a0.counts, so); a.mask = ess_at(a0.mask, so); a.pose = ess_at(a0.pose, so);
    a.result = ess_at(a0.result, (size_t)p * a0.result_stride);
    return a;
}

// the problem of a one-thread-per-problem kernel, -1 for a thread beyond the last
static __device__ __forceinline__ int ess_thread_prob(const EssArgs& a0)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    return p < a0.n_prob ? p : -1;
}

__global__ void k_ess_init(const EssArgs a0)
{
    const EssArgs a = ess_prob(a0, blockIdx.y);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = ess_n(a);
    if (i == 0) {
        EssState& s = *a.state;
        s.rng_state = 0xffffffffffffffffULL;
        s.niters = a.max_iters;
        s.max_good = 0;
        s.best_it = -1; s.best_cand = -1;
        s.iters_run = 0;
        s.done = n <= 5 ? 1 : 0;        // n == 5: no RANSAC (k_ess_five); n < 5: no model
        for (int k = 0; k < 4; k++) s.good4[k] = 0;
    }
    if (i >= n) return;
    const float2 p0 = a.pts0[i], p1 = a.pts1[i];
    const double focal = a.cal->focal, ppx = a.cal->ppx, ppy = a.cal->ppy;
    a.q0[i] = make_double2(((double)p0.x - ppx) / focal, ((double)p0.y - ppy) / focal);
    a.q1[i] = make_double2(((double)p1.x - ppx) / focal, ((double)p1.y - ppy) / focal);
}

__global__ void k_ess_subsets(const EssArgs a0, int it0, int it1)
{
    const int p = ess_thread_prob(a0);
    if (p < 0) return;
    const EssArgs a = ess_prob(a0, p);
    EssState& s = *a.state;
    if (s.done) return;
    const int n = ess_n(a);
    Rng rng(s.rng_state);
    const int last = it1 < s.niters ? it1 : s.niters;
    for (int it = it0; it < last; it++) {
        int idx[5];                     // n > 5 here
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
        for (int i = 0; i < 5; i++) a.subsets[it * 5 + i] = idx[i];
    }
    s.rng_state = rng.state;
}

__global__ void __launch_bounds__(32) k_ess_hypotheses(const EssArgs a0, int it0, int it1)
{
    const EssArgs a = ess_prob(a0, blockIdx.y);
    const int it = it0 + blockIdx.x * blockDim.x + threadIdx.x;
    const EssState& s = *a.state;
    if (s.done || it >= it1 || it >= s.niters) return;
    double q0[10], q1[10];
    for (int i = 0; i < 5; i++) {
        const int j = a.subsets[it * 5 + i];
        const double2 u = a.q0[j], v = a.q1[j];
        q0[2 * i] = u.x; q0[2 * i + 1] = u.y; q1[2 * i] = v.x; q1[2 * i + 1] = v.y;
    }
    a.nmodels[it] = five_point(q0, q1, a.models + (size_t)it * 90);
}

__global__ void __launch_bounds__(128) k_ess_count(const EssArgs a0, int it0, int it1)
{
    const EssArgs a = ess_prob(a0, blockIdx.z);
    const int it = it0 + blockIdx.x, cand = blockIdx.y;
    const EssState& s = *a.state;
    if (s.done || it >= it1 || it >= s.niters) return;
    if (cand >= a.nmodels[it]) return;
    __shared__ double E[9];
    __shared__ int total;
    if (threadIdx.x < 9) E[threadIdx.x] = a.models[(size_t)it * 90 + cand * 9 + threadIdx.x];
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    const int n = ess_n(a);
    const float thr2 = a.cal->thr2;
    int c = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double2 u = a.q0[i], v = a.q1[i];
        c += sampson_err(E, u.x, u.y, v.x, v.y) <= thr2;
    }
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31) == 0) atomicAdd(&total, c);
    __syncthreads();
    if (threadIdx.x == 0) a.counts[it * 10 + cand] = total;
}

__global__ void k_ess_replay(const EssArgs a0, int it0, int it1)
{
    const int p = ess_thread_prob(a0);
    if (p < 0) return;
    const EssArgs a = ess_prob(a0, p);
    EssState& s = *a.state;
    if (s.done) return;
    const int n = ess_n(a);
    int it = it0;
    for (; it < it1 && it < s.niters; it++) {
        const int nm = a.nmodels[it];
        for (int m = 0; m < nm; m++) {
            const int good = a.counts[it * 10 + m];
            if (good > max(s.max_good, 4)) {
                s.best_it = it; s.best_cand = m;
                s.max_good = good;
                s.niters = ransac_update_num_iters(a.prob, (double)(n - good) / n, 5, s.niters);
            }
        }
    }
    s.iters_run = it;
    if (it >= s.niters || it1 >= a.max_iters) s.done = 1;
}

// Exactly five correspondences (= model points): OpenCV runs no RANSAC.  findEssentialMat returns every candidate of one
// five-point solve, stacked (3k x 3), with an all-ones mask; recoverPose only accepts a 3 x 3 E.  So a single candidate is
// the model, with all five points inliers; any other count leaves no model (k_ess_pick reports the reference's abort).
__global__ void k_ess_five(const EssArgs a0)
{
    const int p = ess_thread_prob(a0);
    if (p < 0) return;
    const EssArgs a = ess_prob(a0, p);
    if (ess_n(a) != 5) return;
    EssState& s = *a.state;
    double q0[10], q1[10];
    for (int i = 0; i < 5; i++) {
        q0[2 * i] = a.q0[i].x; q0[2 * i + 1] = a.q0[i].y; q1[2 * i] = a.q1[i].x; q1[2 * i + 1] = a.q1[i].y;
    }
    const int nm = five_point(q0, q1, a.models);
    a.nmodels[0] = nm;
    if (nm == 1) { s.best_it = 0; s.best_cand = 0; s.max_good = 5; }
}

__global__ void k_ess_mask(const EssArgs a0)
{
    const EssArgs a = ess_prob(a0, blockIdx.y);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const EssState& s = *a.state;
    const int n = ess_n(a);
    if (i >= n) return;
    if (s.best_it < 0) { a.mask[i] = 0; return; }
    const double* E = a.models + (size_t)s.best_it * 90 + s.best_cand * 9;
    const double2 u = a.q0[i], v = a.q1[i];
    a.mask[i] = (n == 5 || sampson_err(E, u.x, u.y, v.x, v.y) <= a.cal->thr2) ? 1 : 0;
}

__global__ void k_ess_decompose(const EssArgs a0)
{
    const int p = ess_thread_prob(a0);
    if (p < 0) return;
    const EssArgs a = ess_prob(a0, p);
    const EssState& s = *a.state;
    if (s.best_it < 0) return;
    const double* E = a.models + (size_t)s.best_it * 90 + s.best_cand * 9;
    for (int k = 0; k < 9; k++) a.pose[21 + k] = E[k];
    decompose_essential(E, a.pose, a.pose + 9, a.pose + 18);      // R1 | R2 | t | E
}

__global__ void __launch_bounds__(128) k_ess_cheirality(const EssArgs a0)
{
    const EssArgs a = ess_prob(a0, blockIdx.y);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    EssState& s = *a.state;
    if (s.best_it < 0) return;
    int ok[4] = {0, 0, 0, 0};
    if (i < ess_n(a) && a.mask[i]) {
        const double2 u = a.q0[i], v = a.q1[i];
        const double* t = a.pose + 18;
        const double tn[3] = {-t[0], -t[1], -t[2]};
        ok[0] = cheirality_ok(a.pose, t, u.x, u.y, v.x, v.y, 50.0);
        ok[1] = cheirality_ok(a.pose + 9, t, u.x, u.y, v.x, v.y, 50.0);
        ok[2] = cheirality_ok(a.pose, tn, u.x, u.y, v.x, v.y, 50.0);
        ok[3] = cheirality_ok(a.pose + 9, tn, u.x, u.y, v.x, v.y, 50.0);
    }
    for (int k = 0; k < 4; k++) {
        int c = ok[k];
        for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
        if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s.good4[k], c);
    }
}

__global__ void k_ess_pick(const EssArgs a0)
{
    const int p = ess_thread_prob(a0);
    if (p < 0) return;
    const EssArgs a = ess_prob(a0, p);
    const EssState& s = *a.state;
    EssResult& r = *a.result;
    const int n = ess_n(a);
    r.n_inliers = s.max_good; r.iters = s.iters_run; r.ok = s.best_it >= 0 ? 1 : 0;
    r.n_cand = n == 5 ? a.nmodels[0] : 0;
    r.status = s.best_it >= 0 ? ESS_OK : n < 5 ? ESS_TOO_FEW : n == 5 ? ESS_FIVE_CANDIDATES : ESS_NO_MODEL;
    if (s.best_it < 0) {
        for (int k = 0; k < 9; k++) { r.R[k] = (k % 4 == 0) ? 1.0 : 0.0; r.E[k] = 0.0; }
        r.t[0] = r.t[1] = r.t[2] = 0.0; r.n_good = 0;
        return;
    }
    const int* g = s.good4;
    int k = 3;                                    // recoverPose's order of preference on ties
    if (g[0] >= g[1] && g[0] >= g[2] && g[0] >= g[3]) k = 0;
    else if (g[1] >= g[0] && g[1] >= g[2] && g[1] >= g[3]) k = 1;
    else if (g[2] >= g[0] && g[2] >= g[1] && g[2] >= g[3]) k = 2;
    const double* R = a.pose + ((k & 1) ? 9 : 0);
    const double sgn = k >= 2 ? -1.0 : 1.0;
    for (int j = 0; j < 9; j++) { r.R[j] = R[j]; r.E[j] = a.pose[21 + j]; }
    for (int j = 0; j < 3; j++) r.t[j] = sgn * a.pose[18 + j];
    r.n_good = g[k];
}

static size_t ess_up(size_t x) { return (x + 255) / 256 * 256; }

// one scratch block: normalised points | state | subsets | models | nmodels | counts | mask | pose | result
size_t vo_ess_scratch_bytes(int n_max, int max_iters)
{
    const size_t n = n_max > 0 ? (size_t)n_max : 1, it = (size_t)max_iters;
    return 2 * ess_up(n * sizeof(double2)) + ess_up(sizeof(EssState)) + ess_up(it * 5 * sizeof(int)) +
           ess_up(it * 90 * sizeof(double)) + ess_up(it * sizeof(int)) + ess_up(it * 10 * sizeof(int)) + ess_up(n) +
           ess_up(30 * sizeof(double)) + ess_up(sizeof(EssResult));
}

void vo_ess_bind(EssArgs& a, void* scratch, int n_max, int max_iters)
{
    const size_t n = n_max > 0 ? (size_t)n_max : 1, it = (size_t)max_iters;
    uint8_t* b = (uint8_t*)scratch;
    auto take = [&](size_t bytes) { uint8_t* p = b; b += ess_up(bytes); return p; };
    a.n_max = n_max; a.max_iters = max_iters;
    a.n_prob = 1; a.scratch_stride = 0; a.pts_stride = 0; a.n_stride = 0; a.result_stride = 0; a.cal_stride = 0;
    a.prob = 0.999;
    a.q0 = (double2*)take(n * sizeof(double2)); a.q1 = (double2*)take(n * sizeof(double2));
    a.state = (EssState*)take(sizeof(EssState));
    a.subsets = (int*)take(it * 5 * sizeof(int));
    a.models = (double*)take(it * 90 * sizeof(double));
    a.nmodels = (int*)take(it * sizeof(int));
    a.counts = (int*)take(it * 10 * sizeof(int));
    a.mask = take(n);
    a.pose = (double*)take(30 * sizeof(double));
    a.result = (EssResult*)take(sizeof(EssResult));
}

int vo_launch_essential(const EssArgs& a, cudaStream_t s)
{
    int launches = 0;
    const int np = a.n_prob;
    const int nb = (a.n_max + 127) / 128 > 0 ? (a.n_max + 127) / 128 : 1;
    const int nt = (np + 31) / 32;                       // one thread per problem
    k_ess_init<<<dim3(nb, np), 128, 0, s>>>(a); launches++;
    k_ess_five<<<nt, 32, 0, s>>>(a); launches++;
    const int waves[4] = {0, 32, 128, a.max_iters};
    for (int w = 0; w < 3; w++) {
        const int it0 = waves[w], it1 = waves[w + 1] < a.max_iters ? waves[w + 1] : a.max_iters;
        if (it1 <= it0) break;
        k_ess_subsets<<<nt, 32, 0, s>>>(a, it0, it1);
        k_ess_hypotheses<<<dim3((it1 - it0 + 31) / 32, np), 32, 0, s>>>(a, it0, it1);
        k_ess_count<<<dim3(it1 - it0, 10, np), 128, 0, s>>>(a, it0, it1);
        k_ess_replay<<<nt, 32, 0, s>>>(a, it0, it1);
        launches += 4;
    }
    k_ess_mask<<<dim3(nb, np), 128, 0, s>>>(a);
    k_ess_decompose<<<nt, 32, 0, s>>>(a);
    k_ess_cheirality<<<dim3(nb, np), 128, 0, s>>>(a);
    k_ess_pick<<<nt, 32, 0, s>>>(a);
    return launches + 4;
}
