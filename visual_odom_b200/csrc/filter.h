// filter.h -- launch interface of the ring filter kernel (filter.cu)
#pragma once
#include "common.cuh"

struct FilterArgs {
    int cap;
    size_t call_stride;       // n_units * cap
    const UnitParams* par;    // [units] circ_threshold
    const int* n_pts;         // [units]
    const float2* pts_in;     // [units][cap]           L0
    const float2* pts_out;    // [4][units][cap]        R0, R1, L1, L0_return (ring order)
    const uint8_t* status;    // [4][units][cap]
    const int* ages_in;       // [units][cap] or nullptr
    int* ages_out;            // [units][cap]  (ages+1, compacted by A3 only)
    float2* kept5;            // [5][units][cap]  after A3: L0, R0, L1, R1, L0_return
    int* idx3;                // [units][cap]     original index of A3 survivors
    int* n3;                  // [units]
    float2* valid4;           // [4][units][cap]  after A5/A6: L0, R0, L1, R1
    int* idx5;                // [units][cap]     original index of A5 survivors
    int* n5;                  // [units]
};

cudaError_t vo_launch_ring_filter(const FilterArgs& a, int n_units, cudaStream_t stream);
