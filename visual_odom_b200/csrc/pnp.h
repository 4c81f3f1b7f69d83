// pnp.h -- launch interface of the triangulation and PnP/RANSAC kernels (pnp.cu)
#pragma once
#include "common.cuh"

#define VO_PNP_OK 0
#define VO_PNP_TOO_FEW (-3)            // n < 4: the reference would abort inside cv::solvePnPRansac
#define VO_PNP_NO_MODEL 1              // RANSAC found no model with > 4 inliers: pose = caller's guess

struct PnpState {
    unsigned long long rng_state;
    int niters;       // current adaptive iteration bound
    int max_good;
    int best_it;
    int iters_run;
    int done;
};

struct vo_unit_result_dev {
    int n_features, n_detected, n_tracked, n_valid, n_inliers, ransac_iters, pnp_status, pad_;
    double rvec[3], tvec[3], R[9];
};

struct TriArgs {
    int cap;
    const int* n_pts;        // [units]
    const float2* pts_l;     // [units][cap]
    const float2* pts_r;     // [units][cap]
    float3* X;               // [units][cap]
    float4* X4;              // optional [units][cap]: homogeneous points as cv::triangulatePoints returns them
    const CamCalib* cal;     // [units]: Pl / Pr of each unit
};

struct PnpArgs {
    int n_units, cap;
    int iterations;          // the stride of subsets / models / counts (the largest count); unit u runs par[u].pnp_iterations
    const int* n_pts;        // [units]
    const float3* X;         // [units][cap]
    const float2* x;         // [units][cap]   image points (pointsLeft_t1)
    const CamCalib* cal;     // [units]: fu, fv, uc, vc of each unit
    const UnitParams* par;   // [units]: pnp_iterations, thr2, confidence of each unit
    const double* t_prev;    // [units][3]
    PnpState* state;         // [units]
    int* subsets;            // [units][iterations][5]
    double* models;          // [units][iterations][12]  R (9) + t (3)
    int* counts;             // [units][iterations]
    int* inliers;            // [units][cap]
    vo_unit_result_dev* results;   // [units]
};

int vo_launch_triangulate(const TriArgs& a, int n_units, cudaStream_t stream);
int vo_launch_pnp(const PnpArgs& a, cudaStream_t stream);
