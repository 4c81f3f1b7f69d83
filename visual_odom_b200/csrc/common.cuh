// common.cuh -- shared declarations for the vo_b200 CUDA library (sm_90a only).
//
// Device data layout (see DESIGN.md "Data layout in HBM"):
//   Every pyramid level l of every image lives in ONE allocation per level:
//     u8  image plane  : [n_img][hp_l][pitch_l]      bytes,  origin of pixel (0,0) at (PAD, PAD)
//     s16x2 derivative : [n_img][hp_l][pitch_l]      uint32 (lo16 = dI/dx, hi16 = dI/dy), same origin
//   with hp_l = h_l + 2*PAD, pitch_l = roundup(w_l + 2*PAD, 64).  The u8 border is REFLECT_101
//   filled (what OpenCV's LK pyramid pads with), the derivative border is zero (BORDER_CONSTANT),
//   so the LK kernel needs no border logic and 3-D TMA boxes never leave the allocation.
//   With images of several sizes in one run (PlaneGeom below), w_l / h_l are the envelope: a smaller
//   image's u8 plane is REFLECT_101 padded at its own size over the whole envelope plane, and the
//   derivative pass writes zeros over the envelope area outside the image, so the zero border holds
//   whatever size the plane held before.
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

#define VO_PAD 32            // border (pixels) on every side of every level
#define VO_MAX_LEVELS 8      // pyramid images (maxLevel + 1)
#define VO_WIN 21            // LK window (the reference hard-codes Size(21,21), feature.cpp:127): k_lk_ring's
#define VO_WIN_MIN 3         // vo_params.lk_win range: cv2 asserts winSize > 2; other windows run k_lk_win (lk_win.cu)
#define VO_WIN_MAX 32        // a window of up to VO_PAD pixels reads inside the padded planes
static_assert(VO_WIN_MAX <= VO_PAD, "every window read must stay inside the padding");

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

// One raw image plane's own size, where a run holds images of several sizes (vo_mseq_begin_sized).  The planes are then
// allocated at the envelope (PyrGeom: the largest width and height per level), and the kernels that must see an image's
// own border, raster or bucket grid read its entry of the context's geometry table (ctx.h vo_ctx::d_geo) instead of the
// launch-wide size.  A null table pointer means "every plane is the launch-wide size" (every other path).
struct PlaneGeom {
    int w[VO_MAX_LEVELS], h[VO_MAX_LEVELS];   // image size per pyramid level: level l + 1 is ((w_l + 1) / 2, (h_l + 1) / 2)
    int pitch;                                // raw plane row pitch in bytes (rows are packed: w[0])
    int pad_;
};

// effective pyramid depth (maxLevel + 1) of a w x h image: OpenCV stops adding levels once one is not larger than the
// win x win window
static inline int vo_pyr_depth(int w, int h, int max_level, int win)
{
    int n = 1;
    for (int l = 1; l <= max_level; l++) {
        const int nw = (w + 1) / 2, nh = (h + 1) / 2;
        if (nw <= win || nh <= win) break;
        w = nw; h = nh; n++;
    }
    return n;
}

// One camera as the triangulation, PnP and five-point kernels read it: one entry per buffer unit in the context's
// calibration table (ctx.h vo_ctx::d_cal).  Every value is computed on the host with the expressions of the reference's
// callers (vo_calib_from), so a kernel sees the same bits whichever unit or problem it serves.
struct CamCalib {
    double Pl[12], Pr[12];        // k_triangulate: the float projection matrices widened to double
    double fu, fv, uc, vc;        // PnP: K = P_l(0:3, 0:3) as floats (main.cpp:75 / visualOdometry.cpp:141), widened
    double focal, ppx, ppy;       // five-point branch: `double focal = projMatrl.at<float>(0, 0)`, principle_point
                                  // (visualOdometry.cpp:144-145)
    float thr2;                   // (float)((threshold / focal)^2), threshold 1.0 of the findEssentialMat call (:154)
    int pad_;
};

// One unit's tracking parameters as the kernels read them: one entry per buffer unit in the context's parameter table
// (ctx.h vo_ctx::d_par), beside the unit's calibration entry.  vo_unit_params (ctx.h) computes every value on the host
// with the expressions the launch sites used when the values were launch-wide, so a unit at the context's vo_params sees
// the same bits.
struct UnitParams {
    double eps2;                  // LK: epsilon^2 of the epsilon clamped to [0, 10]
    double confidence;            // PnP: pnp_confidence
    float min_eig;                // LK: lk_min_eig as a float (cv::LKTrackerInvoker keeps minEigThreshold as one)
    float thr2;                   // PnP: (float)((double)pnp_reproj_error^2)
    int max_iters;                // LK: lk_max_iters clamped to [0, 100]
    int pnp_iterations;           // PnP: max(pnp_iterations, 1), at most the context's (the RANSAC scratch)
    int fast_threshold, circ_threshold;
    int refill_threshold, bucket_rows_divisor, features_per_bucket, bucket_age_threshold;   // sequence modes only
};

// the five-point branch's camera values (also vo_mono_rotation's, which takes focal / pp directly)
static inline void vo_calib_set_ess(CamCalib& c, double focal, double ppx, double ppy)
{
    c.focal = focal; c.ppx = ppx; c.ppy = ppy;
    const double thr = 1.0 / focal;                // threshold /= (fx + fy) / 2
    c.thr2 = (float)(thr * thr);
}

// the PnP intrinsics of a float K (row-major 3 x 3)
static inline void vo_calib_set_pnp(CamCalib& c, const float K9[9])
{
    c.fu = (double)K9[0]; c.fv = (double)K9[4]; c.uc = (double)K9[2]; c.vc = (double)K9[5];
}

// every value from one stereo pair of projection matrices (row-major 3 x 4 floats)
static inline CamCalib vo_calib_from(const float P_l[12], const float P_r[12])
{
    CamCalib c;
    for (int k = 0; k < 12; k++) { c.Pl[k] = (double)P_l[k]; c.Pr[k] = (double)P_r[k]; }
    const float K9[9] = {P_l[0], P_l[1], P_l[2], P_l[4], P_l[5], P_l[6], P_l[8], P_l[9], P_l[10]};
    vo_calib_set_pnp(c, K9);
    vo_calib_set_ess(c, (double)P_l[0], (double)P_l[2], (double)P_l[6]);
    c.pad_ = 0;
    return c;
}

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
