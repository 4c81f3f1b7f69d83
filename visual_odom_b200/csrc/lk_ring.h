// lk_ring.h -- launch interface of the LK ring kernel (lk_ring.cu)
#pragma once
#include "common.cuh"

// The kernel is built for 8 persistent CTAs of 2 warps per SM: 128 registers per thread, the whole register file.
#define LK_WARPS_PER_CTA 2
#define LK_CTAS_PER_SM 8

struct LkMaps {
    CUtensorMap img_i[VO_MAX_LEVELS];  // u8 planes, box 48 x 22 x 1 (I window, 16-byte aligned start)
    CUtensorMap img_j[VO_MAX_LEVELS];  // u8 planes, box 48 x 32 x 1 (J tile)
    CUtensorMap der[VO_MAX_LEVELS];    // s16x2 (uint32) planes, box 28 x 22 x 1
};

struct LkArgs {
    int n_units;            // work units in this launch
    int cap;                // feature capacity per unit (stride of the point arrays)
    const int* n_pts;       // [n_units] live feature count per unit (device) or nullptr = cap
    int imgs_per_unit;      // planes per unit in the pyramid (4 for the ring, 2 for a single call)
    int img_plane0;         // absolute plane index of this launch's first unit (unit-range launches)
    int ncalls;             // chained calcOpticalFlowPyrLK calls (4 for the ring)
    int img_prev[4];        // plane index (within the unit) of prev image per call
    int img_next[4];        // plane index of next image per call
    int nlevels;            // pyramid images (effective maxLevel + 1)
    int lw[VO_MAX_LEVELS], lh[VO_MAX_LEVELS];
    const PlaneGeom* geo;   // geometry table indexed by absolute plane (images of several sizes), or nullptr = lw / lh
    const UnitParams* par;  // [n_units] each unit's criteria: max_iters, eps2, min_eig
    const float2* pts_in;   // [n_units][cap]
    float2* pts_out;        // [ncalls][n_units][cap]   (call_stride = n_units*cap)
    uint8_t* status_out;    // [ncalls][n_units][cap]
    float* err_out;         // optional, same shape
    size_t call_stride;
    // work queue of the persistent warps: queue[0] = next item, queue[1] = warps that ran dry (the last one
    // resets both, so the pair is clean for the next launch that uses it); items = n_units * per_unit
    int* queue;
    int per_unit;           // feature slots per unit that can be live (<= cap)
    int span;               // phases (level-solves) per work item; 0 or >= ncalls*nlevels = one item per feature-ring
    int* progress;          // [n_units][cap] phases completed per feature (hand-over between items; all zero between launches)
    // plane geometry per level, for k_lk_win's plain loads (k_lk_ring reads the planes through LkMaps)
    const uint8_t* img_base[VO_MAX_LEVELS];
    const uint32_t* der_base[VO_MAX_LEVELS];
    int pitch[VO_MAX_LEVELS];
    size_t plane[VO_MAX_LEVELS];
};

size_t vo_lk_smem_bytes();
cudaError_t vo_lk_prepare();
// sm_count sizes the persistent grid (CTAs = min(needed, sm_count * LK_CTAS_PER_SM))
cudaError_t vo_launch_lk_ring(const LkMaps& maps, const LkArgs& args, int sm_count, cudaStream_t stream);
// k_lk_win (lk_win.cu): the same ring at a win x win window, VO_WIN_MIN <= win <= VO_WIN_MAX.  It reads the planes with
// plain loads (img_base / der_base / pitch / plane) and runs one work item per feature-ring: span and progress are not
// read
cudaError_t vo_launch_lk_win(const LkArgs& args, int win, int sm_count, cudaStream_t stream);
int vo_launch_pyramid(const PyrGeom& pg, const uint8_t* const* src_tab_dev, int src_pitch, const PlaneGeom* geo, cudaStream_t stream);
