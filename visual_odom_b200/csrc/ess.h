// ess.h -- launch interface of the five-point essential-matrix RANSAC + recoverPose kernels (ess.cu)
#pragma once
#include "common.cuh"

struct EssState {
    unsigned long long rng_state;
    int niters;       // current adaptive iteration bound
    int max_good;
    int best_it, best_cand;
    int iters_run;
    int done;
    int good4[4];     // recoverPose: points in front of both cameras for (R1,t) (R2,t) (R1,-t) (R2,-t)
};

// where the reference aborts (cv::findEssentialMat / cv::recoverPose throw); R = I, t = 0 then
enum EssStatus {
    ESS_OK = 0,
    ESS_TOO_FEW = 1,          // n < 5
    ESS_NO_MODEL = 2,         // no E with more than 4 inliers
    ESS_FIVE_CANDIDATES = 3,  // n == 5 and the one five-point solve gave other than exactly one E
};

struct EssResult {
    double R[9], t[3], E[9];
    int n_inliers, n_good, iters, ok;
    int n_cand;       // n == 5 only: five-point candidates of the one solve (OpenCV returns them all, stacked)
    int status;       // EssStatus
};

struct EssArgs {
    const int* n;             // correspondences (device: the sequence mode's count is only known on the device)
    int n_max;                // host-known bound of *n: sizes the per-point grids and buffers
    int max_iters;            // 1000 (cv::findEssentialMat's default maxIters)
    const float2* pts0;       // pointsLeft_t0
    const float2* pts1;       // pointsLeft_t1
    const CamCalib* cal;      // focal, ppx, ppy, thr2 of the problem's camera
    double prob;              // 0.999
    double2* q0;              // [n_max] normalised points
    double2* q1;
    EssState* state;
    int* subsets;             // [max_iters][5]
    double* models;           // [max_iters][10][9]
    int* nmodels;             // [max_iters]
    int* counts;              // [max_iters][10]
    uint8_t* mask;            // [n_max] inliers of the best E
    double* pose;             // [30] R1 | R2 | t | E of the best model
    EssResult* result;
    // n_prob independent problems in one launch: the pointers above are problem 0's, problem p finds its own `stride`
    // further on (vo_ess_bind sets one problem with zero strides)
    int n_prob;
    size_t scratch_stride;    // bytes, q0 .. pose (one scratch block per problem)
    int pts_stride;           // float2 elements, pts0 / pts1
    int n_stride;             // ints, n
    size_t result_stride;     // bytes, result
    int cal_stride;           // entries, cal
};

#define VO_ESS_ITERS 1000      // cv::findEssentialMat's default maxIters

// bytes of one scratch block for up to n_max points (everything EssArgs points to except pts0 / pts1 / n / cal), and the
// args of one problem laid out over it (prob = 0.999, the literal double of the reference's findEssentialMat call, :154)
size_t vo_ess_scratch_bytes(int n_max, int max_iters);
void vo_ess_bind(EssArgs& a, void* scratch, int n_max, int max_iters);
// A fixed launch sequence whatever each *n turns out to be and whatever n_prob is (graph-capturable, no host sync): per
// problem, n < 5 ends without a model, n == 5 takes k_ess_five, n > 5 the RANSAC waves, which skip themselves once that
// problem's adaptive bound is reached.  Every kernel takes its problem from a grid dimension or, for the per-problem
// bookkeeping, one thread per problem; a problem's arithmetic is that of running it alone.
int vo_launch_essential(const EssArgs& a, cudaStream_t s);
