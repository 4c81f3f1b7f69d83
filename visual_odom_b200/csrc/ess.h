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

struct EssResult {
    double R[9], t[3], E[9];
    int n_inliers, n_good, iters, ok;
    int n_cand;       // n == 5 only: five-point candidates of the one solve (OpenCV returns them all, stacked)
};

struct EssArgs {
    int n;                    // correspondences
    int max_iters;            // 1000 (cv::findEssentialMat's default maxIters)
    const float2* pts0;       // pointsLeft_t0
    const float2* pts1;       // pointsLeft_t1
    double focal, ppx, ppy;   // `double focal = projMatrl.at<float>(0, 0)`, principle_point (visualOdometry.cpp:144-145)
    double prob;              // 0.999
    float thr2;               // (float)((threshold / focal)^2)
    double2* q0;              // [n] normalised points
    double2* q1;
    EssState* state;
    int* subsets;             // [max_iters][5]
    double* models;           // [max_iters][10][9]
    int* nmodels;             // [max_iters]
    int* counts;              // [max_iters][10]
    uint8_t* mask;            // [n] inliers of the best E
    double* pose;             // [30] R1 | R2 | t | E of the best model
    EssResult* result;
};

int vo_launch_essential(const EssArgs& a, cudaStream_t s);
