// common.cuh -- shared declarations for the vo_b200 CUDA library (sm_90a only).
//
// Device data layout (see DESIGN.md "Data layout in HBM"):
//   Every pyramid level l of every image lives in ONE allocation per level:
//     u8  image plane  : [n_img][hp_l][pitch_l]      bytes,  origin of pixel (0,0) at (PAD, PAD)
//     s16x2 derivative : [n_img][hp_l][pitch_l]      uint32 (lo16 = dI/dx, hi16 = dI/dy), same origin
//   with hp_l = h_l + 2*PAD, pitch_l = roundup(w_l + 2*PAD, 64).  The u8 border is REFLECT_101
//   filled (what OpenCV's LK pyramid pads with), the derivative border is zero (BORDER_CONSTANT),
//   so the LK kernel needs no border logic and 3-D TMA boxes never leave the allocation.
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

#define VO_PAD 32            // border (pixels) on every side of every level
#define VO_MAX_LEVELS 8      // pyramid images (maxLevel + 1)
#define VO_WIN 21            // LK window (the reference hard-codes Size(21,21), feature.cpp:127)

struct LevelGeom {
    int w, h;            // image size at this level
    int pitch;           // row pitch in elements (bytes for u8, uint32 for derivative)
    int hp;              // padded height
    uint8_t*  img;       // base of plane 0 (padded origin, NOT pixel (0,0))
    uint32_t* der;       // base of derivative plane 0
    size_t plane;        // pitch*hp, elements per image plane
};

struct PyrGeom {
    int nlevels;
    int n_img;
    LevelGeom lv[VO_MAX_LEVELS];
};

static __host__ __device__ __forceinline__ int vo_reflect101(int p, int len)
{
    if (len == 1) return 0;
    while (p < 0 || p >= len) {
        if (p < 0) p = -p;
        else p = 2 * len - 2 - p;
    }
    return p;
}

#define VO_CUDA_CHECK(expr)                                                             \
    do {                                                                                \
        cudaError_t _e = (expr);                                                        \
        if (_e != cudaSuccess) {                                                        \
            vo_set_error(ctx, "%s:%d CUDA error %s: %s", __FILE__, __LINE__,            \
                         cudaGetErrorName(_e), cudaGetErrorString(_e));                 \
            return VO_E_CUDA;                                                           \
        }                                                                               \
    } while (0)
