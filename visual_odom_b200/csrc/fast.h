// fast.h -- launch interface of the FAST detector kernels (fast.cu)
#pragma once
#include "common.cuh"

struct FastArgs {
    int n_units;
    const uint8_t* const* img_tab;   // device table of raw image pointers
    int img_stride_idx;              // table entries per unit (4); the detector reads entry unit*stride
    int w, h, pitch;                 // raw image geometry
    const UnitParams* par;           // [n_units] fast_threshold
    int nonmax;
    uint8_t* score;                  // [units][h*w]
    size_t score_plane;
    uint16_t* rowbuf;                // [units][h][rowcap] x coordinates per row
    int rowcap;
    int* rowcount;                   // [units][h]
    int* rowoff;                     // [units][h]
    int* n_det;                      // [units] corners found (may exceed corner_cap)
    float2* corners;                 // [units][corner_cap]
    float* resp;                     // optional [units][corner_cap]
    int corner_cap;
    const PlaneGeom* geo;            // geometry table entries of the images, indexed like img_tab (nullptr: all w x h); w / h
                                     // are then the envelope, which lays out score, rowbuf, rowcount and rowoff
};

int vo_launch_fast(const FastArgs& a, cudaStream_t stream);
int vo_launch_select(const float2* corners, int corner_cap, const int* n_det, const int* want, float2* pts, int cap,
                     int* n_pts, int n_units, cudaStream_t stream);
