/*
 * vo_b200.h -- C-ABI of the H100-native visual-odometry front-end (libvo_b200.so).
 *
 * This is the drop-in boundary for the per-frame hot path of ZhenghaoFei/visual_odom:
 * every entry point replaces one OpenCV-backed function of the reference's libfeature /
 * libvisualOdometry shared libraries (reference src/CMakeLists.txt:16-19,31-34).  The C++
 * facade in include/compat/ keeps the reference's own signatures (feature.h, visualOdometry.h)
 * and forwards to these functions; INTEGRATION.md shows the binding.
 *
 * Conventions
 *   - plain C, no torch / OpenCV types; caller owns every buffer; outputs are capacity-passed.
 *   - images are 8-bit single channel (CV_8UC1), row pitch in bytes (reference utils.cpp:179,189).
 *   - points are {float x, y} (cv::Point2f), status is unsigned char, ages are int32.
 *   - every call is synchronous at return unless it says "async" (then it is ordered on the
 *     context's stream; see vo_set_stream / vo_sync).
 *   - return value: VO_OK (0) or a negative VO_E_* code; vo_last_error() gives the text.
 *   - there is NO CPU fallback: if no compute capability 9.0 GPU (H100) is usable, vo_create fails.
 *   - a context is not thread-safe; distinct contexts are independent (one per host thread/GPU).
 */
#ifndef VO_B200_H
#define VO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define VO_API __attribute__((visibility("default")))
#else
#define VO_API
#endif

#define VO_OK 0
#define VO_E_INVALID (-1)        /* bad argument                                             */
#define VO_E_CUDA (-2)           /* CUDA runtime/driver failure (text in vo_last_error)      */
#define VO_E_TOO_FEW_POINTS (-3) /* PnP with < 4 points (the reference aborts in cv::solvePnPRansac) */
#define VO_E_UNSUPPORTED (-4)    /* parameter outside what the kernels are built for         */
/* pnp_status only: RANSAC found no model with more than 4 inliers; the pose is what the reference is left with when it
 * ignores cv::solvePnPRansac's return value: R = I (rvec stays 0), t = the caller's guess */
#define VO_PNP_NO_MODEL 1
#define VO_E_CAPACITY (-5)       /* caller buffer / context capacity too small               */

typedef struct vo_ctx vo_ctx;

typedef struct vo_point2f { float x, y; } vo_point2f;
typedef struct vo_point3f { float x, y, z; } vo_point3f;

/* All literals the reference hard-codes, as run-time parameters (SURVEY.md section 5, "Config").  Away from the
 * reference's values each one does what OpenCV does with it: clamped where OpenCV clamps, refused where it asserts.
 * vo_create sets the context's values.  Every field but lk_win, lk_max_level, fast_nonmax, max_features and max_units
 * can also differ per multi-sequence slot (vo_mseq_params) and per batched unit (vo_batch_params). */
typedef struct vo_params {
    int fast_threshold;      /* 20      reference src/feature.cpp:43; vo_create refuses values
                                        outside [0, 255] (VO_E_INVALID)                           */
    int fast_nonmax;         /* 1       reference src/feature.cpp:44; 0: every FAST corner is kept
                                        with response 0 (as cv::FAST).  Fixed at vo_create: the
                                        corner capacity of a frame depends on it                  */
    int lk_win;              /* 21      reference src/feature.cpp:127 (only 21 is built; vo_create
                                        refuses others with VO_E_UNSUPPORTED)                     */
    int lk_max_level;        /* 3       reference src/feature.cpp:136 (0-based: 4 images); 0..7,
                                        vo_create refuses others (VO_E_UNSUPPORTED).  A pyramid
                                        stops early where a level would not exceed the window     */
    int lk_max_iters;        /* 30      reference src/feature.cpp:128; clamped to [0, 100] as
                                        calcOpticalFlowPyrLK clamps TermCriteria::maxCount        */
    double lk_epsilon;       /* 0.01    reference src/feature.cpp:128; clamped to [0, 10]         */
    double lk_min_eig;       /* 0.001   reference src/feature.cpp:136; used as a float, as
                                        OpenCV's tracker stores and compares it                   */
    int circ_threshold;      /* 0       reference src/visualOdometry.cpp:120; any value (< 0
                                        keeps no point)                                           */
    int pnp_iterations;      /* 500     reference src/visualOdometry.cpp:168; <= 0 runs one
                                        iteration, as cv::solvePnPRansac does                     */
    float pnp_reproj_error;  /* 0.5     reference src/visualOdometry.cpp:169; squared, so a
                                        negative value acts as its magnitude (as in OpenCV)       */
    double pnp_confidence;   /* 0.999   reference src/visualOdometry.cpp:170; vo_create refuses
                                        values outside (0, 1) and NaN (VO_E_INVALID: OpenCV
                                        asserts 0 < confidence < 1)                               */
    int max_features;        /* per-unit feature capacity of the context (default 8192); vo_create
                                refuses values <= 0 (VO_E_INVALID)                                */
    int max_units;           /* work units the batched path can hold at once (default 1)      */
    /* matchingFeatures()' feature bookkeeping (reference src/visualOdometry.cpp:95-107, src/bucket.cpp:16).  Only the
     * sequence modes (vo_seq_*, vo_mseq_*) use them; the batched path (vo_frame_batch, vo_batch_*) selects features by
     * stride and never buckets, so it ignores them.  A multi-sequence slot can have its own (vo_mseq_params).  A sequence mode reads
     * back at most (rows/bs + 1) * (cols/bs + 1) * features_per_bucket points per frame, bs = rows / bucket_rows_divisor
     * (the bucket bound); a begin, open or start whose largest bound exceeds max_features is refused with
     * VO_E_CAPACITY.  These four fields were appended in this order after max_units: callers compiled against a header
     * without them pass a shorter struct and must be rebuilt. */
    int refill_threshold;    /* 2000    reference src/visualOdometry.cpp:95: FAST corners are
                                        appended while the live point count is < refill_threshold
                                        (any value; <= 0 never refills)                           */
    int bucket_rows_divisor; /* 10      reference src/visualOdometry.cpp:106: bucket_size = rows /
                                        bucket_rows_divisor, per sequence from its own rows; vo_create
                                        refuses <= 0 (VO_E_INVALID), a begin / open / start whose
                                        rows / divisor is 0 is refused (VO_E_UNSUPPORTED: the
                                        reference divides by zero)                                */
    int features_per_bucket; /* 1       reference src/visualOdometry.cpp:107 (Bucket(max_size)); vo_create
                                        refuses <= 0 (VO_E_INVALID: the reference reads ages[0] of an
                                        empty bucket)                                             */
    int bucket_age_threshold;/* 10      reference src/bucket.cpp:16: a bucket admits a feature whose
                                        age is < bucket_age_threshold (any value)                 */
} vo_params;

VO_API void vo_default_params(vo_params* p);

/* Create a context on CUDA device `device`.  Fails (VO_E_CUDA) when no GPU is present. */
VO_API int vo_create(int device, const vo_params* params, vo_ctx** out);
VO_API void vo_destroy(vo_ctx* ctx);
VO_API const char* vo_last_error(const vo_ctx* ctx);
/* Run all subsequent work on `cuda_stream` (a cudaStream_t; NULL = the context's own stream). */
VO_API int vo_set_stream(vo_ctx* ctx, void* cuda_stream);
VO_API int vo_sync(vo_ctx* ctx);
/* Number of kernels this context has launched so far (bench.py's "gpu_launches"). */
VO_API long long vo_kernel_launches(const vo_ctx* ctx);
/* Accumulated device time (ms) of the LK ring kernel launches since the last reset,
 * measured with CUDA events on the launching stream; n = launches counted. */
VO_API int vo_lk_kernel_time(vo_ctx* ctx, double* ms_total, long long* n, int reset);
/* Run-time knobs (measurement / debugging): "batch_streams" = 1|2 (unit ranges the batched path runs
 * concurrently, default 2), "lk_staging" = 0 (TMA, default) | 1 (plain loads), "lk_span" = phases (level-solves)
 * per LK work item (0 = automatic, default), "graphs" = 1 (default: kernel sequences on the context's stream, and
 * the two stages of a sequence frame, are replayed as CUDA graphs; unit ranges on the side streams of
 * vo_frame_batch, vo_batch_run and vo_batch_submit are always launched plainly, because their kernels fork to the
 * SM partition or to high-priority helper streams) | 0 (plain launches; needed for vo_lk_kernel_time),
 * "sm_partition" = k > 0: the kernels after the LK ring (filters, triangulation, PnP) of side-stream ranges run on
 * k SMs of their own while FAST, the pyramids and the LK ring share the others | 0: no partition, those kernels run
 * on high-priority helper streams (k < 0 is refused with VO_E_INVALID; without the option the first
 * vo_batch_submit sets aside 8 SMs when the driver supports green contexts), "batch_outputs" = 1: vo_batch_submit
 * also copies the point lists back (vo_batch_outputs), "mono_rotation" = 0 (default) | 1: sequences begun from then
 * on with vo_seq_begin* run trackingFrame2Frame(mono_rotation = true), see vo_seq_wait_mono (a sequence keeps the value
 * it was begun with; vo_mseq_begin* refuse the option, they take the flag VO_MSEQ_MONO_ROTATION instead). */
VO_API int vo_set_option(vo_ctx* ctx, const char* key, double value);

/* ---- A1: cv::FAST(image, kps, threshold, nonmax) + KeyPoint::convert ------------------------
 * replaces featureDetectionFast(), reference src/feature.cpp:39-47 (decl feature.h:48).
 * Output in raster order (y, then x), integer coordinates as float.  *n_out is the number of
 * corners found; at most `cap` are written (VO_E_CAPACITY if n_out > cap, buffer still filled). */
VO_API int vo_fast_detect(vo_ctx* ctx, const uint8_t* img, int w, int h, size_t pitch,
                          vo_point2f* out, float* response /* optional */, int cap, int* n_out);

/* ---- one cv::calcOpticalFlowPyrLK call ---------------------------------------------------------
 * replaces the call inside featureTracking(), reference src/feature.cpp:72 (decl feature.h:52),
 * and is the unit the ring below chains.  err may be NULL. */
VO_API int vo_lk_track(vo_ctx* ctx, const uint8_t* prev, const uint8_t* next, int w, int h, size_t pitch,
                       const vo_point2f* prev_pts, int n, vo_point2f* next_pts, uint8_t* status, float* err);

/* ---- A2 + A3: circularMatching() ---------------------------------------------------------------
 * replaces circularMatching(), reference src/feature.cpp:118-148 (decl feature.h:61-65), i.e. the
 * four chained LK calls L0->R0->R1->L1->L0 and deleteUnmatchFeaturesCircle() (src/feature.cpp:76-116).
 *   pts_l0[n]            input features (points_l_0)
 *   ages_io[n]           in: current_features.ages; out: ages+1, compacted to *n_kept (may be NULL)
 *   o_l0,o_r0,o_l1,o_r1,o_l0_ret  capacity n each: the five point vectors after the erase loop
 *   status4              optional, 4*n bytes: raw status of the four calls, original indexing
 *   raw4                 optional, 4*n points: raw outputs of the four calls (R0,R1,L1,L0_ret), original indexing
 *   kept_idx[n]          original indices of the survivors, ascending; *n_kept their count */
VO_API int vo_circular_match(vo_ctx* ctx, const uint8_t* l0, const uint8_t* r0, const uint8_t* l1,
                             const uint8_t* r1, int w, int h, size_t pitch, const vo_point2f* pts_l0, int n,
                             int32_t* ages_io, vo_point2f* o_l0, vo_point2f* o_r0, vo_point2f* o_l1,
                             vo_point2f* o_r1, vo_point2f* o_l0_ret, uint8_t* status4, vo_point2f* raw4,
                             int32_t* kept_idx, int* n_kept);

/* ---- A8: cv::triangulatePoints + cv::convertPointsFromHomogeneous ------------------------------
 * replaces the call site reference src/main.cpp:170-171 (and Frame::triangulateFeaturePoints,
 * src/Frame.cpp:25-28).  P_l, P_r: row-major 3x4 float (CV_32F, main.cpp:73-74). */
VO_API int vo_triangulate(vo_ctx* ctx, const float P_l[12], const float P_r[12], const vo_point2f* pts_l,
                          const vo_point2f* pts_r, int n, vo_point3f* X);
/* The same triangulation, returned the way cv::triangulatePoints itself returns it (Frame::triangulateFeaturePoints,
 * reference src/Frame.cpp:25-28): X4 = n x 4 floats, point i = the unit-norm homogeneous vector (x, y, z, w) that is
 * column i of OpenCV's 4 x N CV_32F output (same bits, same sign). */
VO_API int vo_triangulate_homogeneous(vo_ctx* ctx, const float P_l[12], const float P_r[12], const vo_point2f* pts_l,
                                      const vo_point2f* pts_r, int n, float* X4);

/* ---- A9: cv::solvePnPRansac(..., SOLVEPNP_ITERATIVE, useExtrinsicGuess) + cv::Rodrigues --------
 * replaces the pose solve of trackingFrame2Frame(), reference src/visualOdometry.cpp:161-189.
 *   K            row-major 3x3 float intrinsics (built from P_l, visualOdometry.cpp:163-165)
 *   rvec_io      in: initial rvec (the reference resets it to 0 every call, :162); out: solution
 *   tvec_io      in: extrinsic guess (previous translation, main.cpp:82,181); out: solution
 *   inliers[n]   ascending inlier indices (CV_32S column in the reference), *n_inliers their count
 *   R_out        row-major 3x3 double = Rodrigues(rvec)
 * n == 4: as OpenCV, no RANSAC: the P3P pose of the first three points that reprojects the fourth best, unrefined, all
 * four reported as inliers, *ransac_iters = 0 (agrees with cv2 to <= 1e-6 on [R|t] in generic scenes; csrc/p3p_math.cuh).
 * Returns VO_E_TOO_FEW_POINTS for n < 4 (the reference would abort with cv::Exception). */
VO_API int vo_pnp_ransac(vo_ctx* ctx, const vo_point3f* X, const vo_point2f* x, int n, const float K[9],
                         double rvec_io[3], double tvec_io[3], int32_t* inliers, int* n_inliers,
                         double R_out[9], int* ransac_iters /* optional */);

/* ---- N5: the mono_rotation = true branch of trackingFrame2Frame (the header default of the reference's flag) -------
 * replaces reference src/visualOdometry.cpp:146-157:
 *     E = cv::findEssentialMat(pointsLeft_t0, pointsLeft_t1, focal, pp, cv::RANSAC, 0.999, 1.0, mask);
 *     cv::recoverPose(E, pointsLeft_t0, pointsLeft_t1, rotation, translation_mono, focal, pp, mask);
 * Five-point RANSAC (1000 iterations at most, adaptive bound) + the four-way cheirality vote.  R_out = `rotation`
 * (row-major 3x3); mask_out (optional, n bytes) = inliers of the best E; *n_inliers their count.
 * n < 5 or no model: VO_E_TOO_FEW_POINTS (OpenCV throws in both cases). */
VO_API int vo_mono_rotation(vo_ctx* ctx, const vo_point2f* pts_t0, const vo_point2f* pts_t1, int n, double focal, double ppx,
                            double ppy, double R_out[9], uint8_t* mask_out, int* n_inliers, int* ransac_iters);

/* ---- batched whole-path API (configs 4/5 of BASELINE.json, bench.py, multi-GPU sharding) ------
 * One work unit = one stereo pair-of-pairs + its feature list (SURVEY.md section 8d "Work unit").
 * The batched path keeps everything device-resident between stages:
 *   FAST on l0 (when pts == NULL) -> even-stride selection of select_n corners
 *   -> pyramids -> LK ring -> status/negative/circular filters -> triangulation -> PnP/RANSAC. */
typedef struct vo_unit {
    const uint8_t *l0, *r0, *l1, *r1;   /* HOST images (w x h, pitch); see vo_batch_submit_device    */
    const vo_point2f* pts;              /* HOST features of l0, or NULL = detect on the GPU         */
    int n_pts;                          /* features in pts; with pts==NULL: number to select        */
    double t_prev[3];                   /* extrinsic guess for the pose solve                       */
} vo_unit;

typedef struct vo_unit_result {
    int n_features;      /* features fed to the ring                                   */
    int n_detected;      /* FAST corners found on l0 (0 when pts were given); in the
                            sequence modes whether or not they were appended (a frame
                            with refill_threshold or more live points appends none)     */
    int n_tracked;       /* survivors of deleteUnmatchFeaturesCircle (A3)              */
    int n_valid;         /* survivors of checkValidMatch/removeInvalidPoints (A5/A6)   */
    int n_inliers;       /* RANSAC inliers                                             */
    int ransac_iters;    /* iterations the adaptive loop ran                           */
    int pnp_status;      /* VO_OK, VO_PNP_NO_MODEL or VO_E_TOO_FEW_POINTS (n < 4); n == 4 runs OpenCV's P3P case, n == 5 one
                            unrefined EPnP on all five (no RANSAC, ransac_iters 0, VO_OK even for a non-finite pose) */
    double rvec[3], tvec[3], R[9];
} vo_unit_result;

/* Allocate/resize the device-resident batch state for n_units units of w x h images; every unit gets the calibration
 * P_l / P_r.  Image size and feature capacity are per context: group rigs with different image sizes by context. */
VO_API int vo_batch_configure(vo_ctx* ctx, int w, int h, int n_units, const float P_l[12], const float P_r[12]);
/* Units [first_unit, first_unit + n_units) get their own calibrations: unit first_unit + i runs its triangulation and PnP
 * with P_l + 12 i / P_r + 12 i (n_units row-major 3 x 4 matrices each), e.g. one context for several stereo rigs of one
 * image size.  A unit keeps its calibration across submissions until it is set again (vo_batch_configure sets every
 * unit); each unit's results are those of a context configured with its calibration alone, bit for bit.  Refused
 * (VO_E_INVALID): a range outside the configured units, NULL matrices, or a call while submissions are in flight
 * (vo_batch_wait them first); like vo_batch_configure it ends an idle sequence-mode run. */
VO_API int vo_batch_calibrate(vo_ctx* ctx, int first_unit, int n_units, const float* P_l, const float* P_r);
/* Units [first_unit, first_unit + n_units) get their own tracking parameters: unit first_unit + i runs with p[i] (NULL p:
 * the context's).  The batched path reads fast_threshold, the LK criteria, circ_threshold and the three PnP fields; the
 * four bookkeeping fields are ignored, as for the context.  A unit keeps its parameters until they are set again
 * (vo_batch_configure resets every unit to the context's); each unit's results are those of vo_frame_batch in a context
 * created with its parameters, bit for bit.  Refused, changing nothing: the range and in-flight rules of
 * vo_batch_calibrate (VO_E_INVALID); an entry that vo_create would refuse (its code and message); lk_win, lk_max_level
 * or fast_nonmax other than the context's (VO_E_UNSUPPORTED); pnp_iterations above the context's (VO_E_CAPACITY: the
 * RANSAC scratch is sized for it).  Like vo_batch_calibrate it ends an idle sequence-mode run. */
VO_API int vo_batch_params(vo_ctx* ctx, int first_unit, int n_units, const vo_params* p);
/* async: copy the units' images (and features) host->device on the context's stream. */
VO_API int vo_batch_upload(vo_ctx* ctx, const vo_unit* units, int n_units, size_t pitch);
/* async: run the whole path for the uploaded units. */
VO_API int vo_batch_run(vo_ctx* ctx);
/* async D2H of the per-unit result records into pinned staging + sync + copy to `results`. */
VO_API int vo_batch_download(vo_ctx* ctx, vo_unit_result* results, int n_units);
/* upload + run + download in one call: the end-to-end entry point. */
VO_API int vo_frame_batch(vo_ctx* ctx, const vo_unit* units, int n_units, size_t pitch, vo_unit_result* results);
/* Pipelined form of vo_frame_batch.  vo_batch_submit fills the resident unit slots [first_unit, first_unit + n_units)
 * from units[0 .. n_units) (units == NULL: re-run what is resident there), runs the whole path on them and stages their
 * result records, all asynchronously; vo_batch_wait blocks until that submission is done and copies the records out.
 * Submissions on disjoint slot ranges overlap on the GPU (H2D and the latency-bound PnP tail of one under the LK ring of
 * the other).  The library runs up to three submissions concurrently (three lanes of streams): with inputs resident on
 * the device two in flight saturate the GPU; with inputs coming from the host configure 3 x B units and keep three
 * submissions of B in flight, so that the upload of step s+2 is already queued while the host reads step s (otherwise the
 * host's enqueue time and the H2D copy sit between two steps of the GPU).  The host images of a submission
 * must stay valid (and, for a true async copy, be pinned) until it has been waited for; a slot range must be waited
 * for before it is submitted again.  vo_batch_fetch of a waited slot is valid until that slot is resubmitted. */
VO_API int vo_batch_submit(vo_ctx* ctx, const vo_unit* units, int first_unit, int n_units, size_t pitch);
VO_API int vo_batch_wait(vo_ctx* ctx, int first_unit, int n_units, vo_unit_result* results);
/* Fetch the per-unit arrays of the last run (any pointer may be NULL). Capacity = max_features.
 *   pts4: 4 x n_valid points (L0,R0,L1,R1 after A6);  kept_idx: n_valid original indices;
 *   X: n_valid 3-D points;  inliers: n_inliers indices into the n_valid list. */
/* With vo_set_option(ctx, "batch_outputs", 1) every submission also returns what the reference's matchingFeatures() /
 * trackingFrame2Frame() hand back (reference src/visualOdometry.h:27-42): the four point lists, the tracked-feature
 * indices, points3D and the inlier list of every unit, packed on the device and copied with ONE device-to-host copy per
 * submission into pinned staging.  vo_batch_outputs reads a waited unit from that staging (layout as vo_batch_fetch;
 * any pointer may be NULL) until its slot is resubmitted, whatever feature counts other slot ranges are submitted with;
 * *d2h_bytes_per_unit = bytes that cross PCIe per unit (a block sized for the largest feature count of the resident slots). */
VO_API int vo_batch_outputs(vo_ctx* ctx, int unit, vo_point2f* pts4, int32_t* kept_idx, vo_point3f* X, int32_t* inliers,
                            size_t* d2h_bytes_per_unit);
VO_API int vo_batch_fetch(vo_ctx* ctx, int unit, vo_point2f* pts_in, vo_point2f* pts4, int32_t* kept_idx,
                          vo_point3f* X, int32_t* inliers);

/* ---- images already in device memory (sequence and batched modes) ----------------------------------------------------
 * One caller-owned image in device memory of the context's GPU (cudaMalloc'ed or managed; host and pinned-host memory
 * are refused).  Pixel (x, y), channel c is read at data + y * row_pitch + x * pixel_stride + c * channel_stride, at
 * any alignment:
 *   gray (H, W)            pixel_stride 1, row_pitch >= W
 *   interleaved (H, W, 3)  pixel_stride 3, channel_stride 1      (cv::Mat CV_8UC3, torch HWC)
 *   planar (3, H, W)       pixel_stride 1, channel_stride = plane size (torch CHW, e.g. torchvision's CUDA decoders)
 * Colour is converted exactly as cv::cvtColor(BGR2GRAY / RGB2GRAY): (b*3735 + g*19235 + r*9798 + 2^14) >> 15.
 * Refused (VO_E_INVALID): a pointer that is not device memory of the context's GPU, pixel_stride < 1,
 * row_pitch < w * pixel_stride, channel_stride < 1 for colour, an unknown format. */
#define VO_FMT_GRAY 0
#define VO_FMT_BGR  1
#define VO_FMT_RGB  2
typedef struct vo_dimage {
    const uint8_t* data;    /* device pointer to pixel (0,0), first channel                                   */
    size_t row_pitch;       /* bytes between rows                                                               */
    int    pixel_stride;    /* bytes between horizontally adjacent pixels (1: gray / planar, 3: interleaved)    */
    size_t channel_stride;  /* bytes between a pixel's channels (1: interleaved HWC, plane size: planar CHW);    */
                            /* ignored for VO_FMT_GRAY                                                          */
    int    format;          /* VO_FMT_*                                                                         */
} vo_dimage;
/* vo_unit with device images in place of the four host pointers and the pitch; pts stays a HOST list (or NULL). */
typedef struct vo_dunit {
    vo_dimage l0, r0, l1, r1;
    const vo_point2f* pts;
    int n_pts;
    double t_prev[3];
} vo_dunit;
/* Stream contract of the *_device calls (the rule a PyTorch operation follows; no stream argument, see vo_set_stream):
 *   - the images are read after all work enqueued on the context's stream before the call;
 *   - work enqueued on that stream after the call returns is ordered after the library's last read of the images, so the
 *     caller may overwrite or free them stream-ordered without waiting for results.
 * Every other rule of the host-memory form applies unchanged (frames in flight, slot overlap, mixing of entry points).
 *   vo_seq_begin_device / vo_seq_submit_device   vo_seq_begin / vo_seq_submit; results through vo_seq_wait[_mono]
 *                                                (a push is submit + wait).  The conversion runs on the sequence's copy
 *                                                stream, straight into the image ring, under the previous frame.
 *   vo_batch_submit_device                       vo_batch_submit; results through vo_batch_wait / vo_batch_outputs /
 *                                                vo_batch_fetch.  units == NULL re-runs what is resident, as there. */
VO_API int vo_seq_begin_device(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const vo_dimage* left0,
                               const vo_dimage* right0);
VO_API int vo_seq_submit_device(vo_ctx* ctx, const vo_dimage* left1, const vo_dimage* right1);
VO_API int vo_batch_submit_device(vo_ctx* ctx, const vo_dunit* units, int first_unit, int n_units);

/* ---- multi-GPU: gather of the result records over NCCL (SURVEY.md 8e; one process per GPU, units sharded) -----------
 * The path has no data-path collective; the only exchange is the gather of the fixed-size records.  NCCL is resolved with
 * dlopen at vo_dist_init (VO_E_UNSUPPORTED when the host has none).  Rank 0 makes the id with vo_dist_unique_id and hands the
 * 128 bytes to the other ranks out of band; every rank calls vo_dist_init once.  vo_dist_gather_post posts, without
 * blocking, the records of resident slots [first_unit, first_unit + n_units) (same n_units on every rank): the post is a
 * device-side snapshot, so the slots may be refilled at once and a later submission never waits for another rank.  The
 * exchange itself is batched: one in-place ncclAllGather + one copy into pinned staging per 4 posts, or as soon as
 * vo_dist_gather_wait needs a posted step that has not been exchanged yet.  Up to VO_DIST_DEPTH posts may be outstanding
 * (ranks may drift apart by that many steps before anyone blocks); vo_dist_gather_wait returns the oldest one:
 * all[r * n_units + i] = record i of rank r.  Every rank must post and wait in the same order. */
#define VO_DIST_DEPTH 8
VO_API int vo_dist_unique_id(uint8_t id_out[128]);
VO_API int vo_dist_init(vo_ctx* ctx, const uint8_t id[128], int rank, int world);
VO_API int vo_dist_gather_post(vo_ctx* ctx, int first_unit, int n_units);
VO_API int vo_dist_gather_wait(vo_ctx* ctx, vo_unit_result* all, int cap_records, int* n_records);

/* ---- streaming sequence mode (SURVEY.md 8f, row N1) ------------------------------------------------
 * The state of the reference's main loop (src/main.cpp:87-92,123-181: currentVOFeatures, the previous
 * stereo pair, `translation`) lives on the device.  vo_seq_begin uploads the first pair; each vo_seq_push
 * uploads only the NEW pair, builds only its two pyramids and runs matchingFeatures() (FAST refill,
 * bucketing rows/10 x 1, circular matching, 1-px round-trip check) -> triangulation ->
 * trackingFrame2Frame(mono_rotation=false, or true with the option "mono_rotation", see vo_seq_wait_mono), carrying
 * features / ages / translation to the next frame exactly as the reference does (including the ages-vs-points length
 * skew, SURVEY.md Appendix A item 8).
 *   out      counts + pose of this frame pair
 *   pts4     optional: 4 arrays of pts_cap points (L0, R0, L1, R1 after the circular check); the first
 *            out->n_valid entries of each are meaningful, the rest of the arrays is scratch
 * The per-frame kernel sequence is replayed as two CUDA graphs (front half / pose solve; option "graphs").
 * vo_seq_begin* and vo_mseq_begin* are refused (VO_E_INVALID) while a vo_batch_submit submission has not been waited for,
 * before they change anything: a sequence reuses the buffers and the pinned staging that submission still uses. */
VO_API int vo_seq_begin(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const uint8_t* left0,
                        const uint8_t* right0, size_t pitch);
VO_API int vo_seq_push(vo_ctx* ctx, const uint8_t* left1, const uint8_t* right1, size_t pitch, vo_unit_result* out,
                       vo_point2f* pts4, int pts_cap);
/* same, for inputs with `channels` interleaved bytes per pixel: 1 = gray, 3 = BGR as cv::imread(IMREAD_COLOR) returns
 * it -- the BGR bytes are uploaded as they are and converted on the device with cv::cvtColor(BGR2GRAY)'s fixed-point
 * formula (reference src/utils.cpp:178-179,188-189) inside the frame's graph. */
VO_API int vo_seq_begin_ex(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const uint8_t* left0,
                           const uint8_t* right0, size_t pitch, int channels);
VO_API int vo_seq_push_ex(vo_ctx* ctx, const uint8_t* left1, const uint8_t* right1, size_t pitch, int channels,
                          vo_unit_result* out, vo_point2f* pts4, int pts_cap);
/* Pipelined form: vo_seq_submit enqueues a frame and returns; vo_seq_wait blocks for the OLDEST frame in flight and
 * returns its record (and integrates frame_pose).  At most two frames may be in flight: only the pose solve of frame
 * k+1 depends on the pose solve of frame k (the extrinsic guess), so the upload, pyramids, FAST, bucketing, LK ring,
 * filters and triangulation of frame k+1 run under the latency-bound PnP of frame k -- one frame of result lag buys
 * ~1.7x the frame rate.  Results are identical to vo_seq_push (= submit + wait).  The host images of a submitted frame
 * must stay valid until the call returns for pageable memory, until its vo_seq_wait for pinned memory. */
VO_API int vo_seq_submit(vo_ctx* ctx, const uint8_t* left1, const uint8_t* right1, size_t pitch, int channels);
VO_API int vo_seq_wait(vo_ctx* ctx, vo_unit_result* out, vo_point2f* pts4, int pts_cap);
/* trackingFrame2Frame(..., mono_rotation = true), the reference's header default (src/visualOdometry.h:42), in the sequence
 * mode: set vo_set_option(ctx, "mono_rotation", 1) before vo_seq_begin[_ex].  Each frame then also runs
 *     E = cv::findEssentialMat(pointsLeft_t0, pointsLeft_t1, focal, pp, cv::RANSAC, 0.999, 1.0, mask);
 *     cv::recoverPose(E, pointsLeft_t0, pointsLeft_t1, rotation, translation_mono, focal, pp, mask);
 * (reference src/visualOdometry.cpp:146-157; focal / pp = the float entries of P_l), and the PnP supplies only
 * `translation` (:186-189).  The record's R is recoverPose's rotation; rvec, tvec, n_inliers, ransac_iters and pnp_status
 * stay the PnP's (the same bits as without the option), and the carried translation is the PnP's.  frame_pose integrates
 * (R, tvec) under the main loop's gates.  Where the reference would abort in the branch (fewer than 5 points, no E with
 * more than 4 inliers, exactly 5 points with other than one five-point candidate) the frame is reported with
 * mono.status = VO_E_TOO_FEW_POINTS and R = I, is not integrated, and the sequence goes on -- as a frame whose PnP had
 * fewer than 4 points.  vo_seq_push / vo_seq_wait work on such a sequence too (R = the mono rotation); vo_seq_wait_mono
 * is vo_seq_wait plus the branch's details of the same frame:
 *   mono      the recoverPose result
 *   ess_mask  optional, mask_cap bytes: the essential inlier mask, aligned with the frame's point lists (first
 *             out->n_valid entries meaningful)
 * VO_E_INVALID when the sequence was begun without "mono_rotation". */
typedef struct vo_mono_result {
    int status;        /* VO_OK, or VO_E_TOO_FEW_POINTS where cv::findEssentialMat / cv::recoverPose would throw */
    int n_inliers;     /* essential-matrix RANSAC inliers (the mask's count) */
    int ransac_iters;
    int n_good;        /* recoverPose's return value: inliers in front of both cameras for the chosen pose */
    double R[9];       /* recoverPose rotation (row-major) */
    double t[3];       /* translation_mono (unused by the reference, returned for completeness) */
} vo_mono_result;
VO_API int vo_seq_wait_mono(vo_ctx* ctx, vo_unit_result* out, vo_mono_result* mono, uint8_t* ess_mask, int mask_cap,
                            vo_point2f* pts4, int pts_cap);
/* currentVOFeatures (points / ages may differ in length) and the carried translation (waits for frames in flight) */
VO_API int vo_seq_state(vo_ctx* ctx, vo_point2f* points, int32_t* ages, int cap, int* n_points, int* n_ages, double t_out[3]);

/* ---- several independent sequences through the streaming sequence mode ----------------------------------------------
 * n_seq sequences, each with its own calibration (vo_mseq_begin_calib) or all with one, and each with its own image size
 * (vo_mseq_begin_sized) or all with one, advance in lockstep, one frame each per submission, through the
 * stages of the sequence mode above; every stage is ONE kernel launch for all of them, so a submission costs the launches
 * of one vo_seq_submit whatever n_seq is.  Each sequence's records, point lists, carried state and frame_pose are those of
 * running it alone through vo_seq_begin / vo_seq_push (the same kernels on its own units), bit for bit.
 *   vo_mseq_begin   starts n_seq sequences from their first pairs left0[q] / right0[q] (channels 1 = gray, 3 = BGR, as
 *                   vo_seq_begin_ex; one pitch for all images)
 *   vo_mseq_submit  asynchronous: advances every live sequence by one frame.  left1[q] == right1[q] == NULL retires
 *                   sequence q for the rest of the run (sequences of unequal length): its state and frame_pose freeze and
 *                   its units do no tracking or pose work from then on.  At most two submissions may be in flight, as with
 *                   vo_seq_submit (the front stage of submission k+1 runs under the pose solve of submission k).
 *   vo_mseq_wait    waits for the oldest submission: out[q] as vo_seq_wait's record, status[q] = VO_OK, VO_E_CAPACITY
 *                   (that sequence's glue capacity bits, see vo_last_error) or VO_MSEQ_RETIRED (out[q] zeroed), and
 *                   frame_pose of each live sequence integrated under the main loop's gates.  pts4 is optional:
 *                   n_seq x 4 x pts_cap points, the four lists of sequence q from pts4 + 4 * pts_cap * q.  Returns
 *                   VO_E_CAPACITY when a status is, else VO_OK; every record is filled either way.
 *   vo_mseq_pose / vo_mseq_state   vo_seq_pose / vo_seq_state of sequence q
 * Refused with VO_E_INVALID: n_seq < 1, a third submission in flight, a wait with nothing in flight, a pair with one NULL
 * image, a pair for a retired sequence, unknown flag bits.  VO_E_UNSUPPORTED: the option "mono_rotation" is on (in this
 * mode the branch is asked for with the flag below, for every sequence at once).  VO_E_CAPACITY: n_seq above VO_MSEQ_MAX.
 * Frames already in device memory: vo_mseq_begin_device / vo_mseq_submit_device below.
 * trackingFrame2Frame(mono_rotation = true) for every sequence: vo_mseq_begin_ex with the flag VO_MSEQ_MONO_ROTATION
 * (vo_mseq_begin is vo_mseq_begin_ex with flags = 0).  Each sequence then gets what vo_seq_wait_mono gives a single
 * sequence begun with the option "mono_rotation" -- the record's R is recoverPose's rotation, rvec / tvec / n_inliers /
 * ransac_iters / pnp_status and the carried translation stay the PnP's, a frame where the reference would throw is
 * reported with mono.status = VO_E_TOO_FEW_POINTS and R = I and is not integrated -- bit for bit as running it alone.
 * The essential-matrix RANSAC of all sequences runs as one launch per stage, so the launches per submission stay those
 * of one vo_seq_submit with the option.  Device scratch: about 0.8 MB per sequence and frame in flight at 1241x376.
 *   vo_mseq_wait_mono  vo_mseq_wait plus, per sequence q, mono[q] (zeroed for a retired sequence) and, optionally, the
 *                      essential inlier mask at ess_mask + mask_cap * q, aligned with sequence q's point lists (the first
 *                      out[q].n_valid entries meaningful).  VO_E_INVALID on sequences begun without the flag.
 *                      vo_mseq_wait works on flagged sequences too (R = the mono rotation).
 * Starting either sequence mode ends the other one if it is idle and is refused while it has frames in flight; the
 * vo_seq_* frame calls are refused while vo_mseq_* sequences run and the other way round.  Every other entry point that
 * reuses the shared buffers is refused while submissions are in flight, as for vo_seq_submit. */
#define VO_MSEQ_MAX 64
#define VO_MSEQ_RETIRED 2        /* vo_mseq_wait status: the sequence was retired by this or an earlier submission */
#define VO_MSEQ_MONO_ROTATION 1  /* vo_mseq_begin_ex flag: every sequence runs trackingFrame2Frame(mono_rotation = true) */
VO_API int vo_mseq_begin(vo_ctx* ctx, int n_seq, int w, int h, const float P_l[12], const float P_r[12], const uint8_t* const* left0,
                         const uint8_t* const* right0, size_t pitch, int channels);
VO_API int vo_mseq_begin_ex(vo_ctx* ctx, int n_seq, int w, int h, const float P_l[12], const float P_r[12],
                            const uint8_t* const* left0, const uint8_t* const* right0, size_t pitch, int channels, int flags);
/* vo_mseq_begin_ex with one calibration per sequence: P_l / P_r hold n_seq row-major 3 x 4 matrices each, and sequence q
 * runs with P_l + 12 q / P_r + 12 q, as the reference's main() builds them from its own calibration file
 * (src/main.cpp:67-74).  With VO_MSEQ_MONO_ROTATION each sequence's focal / principal point come from its own P_l.
 * Each sequence's results are those of running it alone through vo_seq_begin with its matrices, bit for bit, and a
 * submission costs the same launches as with one calibration.  vo_mseq_begin_ex is this call with its matrices repeated. */
VO_API int vo_mseq_begin_calib(vo_ctx* ctx, int n_seq, int w, int h, const float* P_l, const float* P_r,
                               const uint8_t* const* left0, const uint8_t* const* right0, size_t pitch, int channels, int flags);
/* vo_mseq_begin_calib with one image size and one row pitch per sequence: sequence q is w[q] x h[q], its images are read
 * pitch[q] bytes per row.  Each sequence's results are those of vo_seq_begin at its own size and calibration, bit for bit
 * (its own pyramid borders, FAST raster, LK image bounds and rows/10 bucket grid), and a submission costs the same launches
 * as with one size.  The image planes are allocated at the envelope of the sizes (the largest width, the largest height),
 * so a later run whose sizes have the same envelope reuses them, and the frame graphs of any earlier run with the same
 * largest rows/10 bucket grid.  vo_mseq_begin_calib is this call
 * with w / h / pitch repeated.  Refused with VO_E_INVALID: NULL w, h or pitch, a size <= 0, pitch[q] < channels * w[q]
 * (and every refusal of vo_mseq_begin_calib); VO_E_UNSUPPORTED: h[q] / 10 == 0, or sizes with different pyramid depths
 * (every size above about 170 pixels on each side has the full depth of lk_max_level = 3).  A refusal changes nothing. */
VO_API int vo_mseq_begin_sized(vo_ctx* ctx, int n_seq, const int* w, const int* h, const float* P_l, const float* P_r,
                               const uint8_t* const* left0, const uint8_t* const* right0, const size_t* pitch,
                               int channels, int flags);
/* Slots [first_slot, first_slot + n) get their own tracking parameters: slot first_slot + i gets p[i] (NULL p: the
 * context's again).  A slot keeps its setting until it is set again.  Every begin call (vo_mseq_begin*,
 * vo_mseq_begin_device), vo_mseq_open and every start reads the setting of each slot it begins, opens or starts; a
 * running sequence keeps the values it began with.  The call changes host state only, so it may be made while frames
 * are in flight.  Each sequence's results are those of a context created with its slot's parameters running it alone,
 * bit for bit, and a submission costs the same launches.  The begin, open and start checks of the bucket bound (rows /
 * bucket_rows_divisor == 0: VO_E_UNSUPPORTED; a bound above max_features: VO_E_CAPACITY) use each slot's own fields.
 * Refused, changing nothing: a range outside 0 .. VO_MSEQ_MAX (VO_E_INVALID); an entry that vo_create would refuse (its
 * code and message); lk_win, lk_max_level or fast_nonmax other than the context's (VO_E_UNSUPPORTED); pnp_iterations
 * above the context's (VO_E_CAPACITY: the RANSAC scratch is sized for it).  max_features and max_units are not read. */
VO_API int vo_mseq_params(vo_ctx* ctx, int first_slot, int n, const vo_params* p);
/* vo_mseq_submit with one row pitch per sequence (pitch[q] is not read for a retiring sequence); vo_mseq_submit is this
 * call with its pitch repeated, so with several sizes it needs a pitch that covers every live sequence's width. */
VO_API int vo_mseq_submit(vo_ctx* ctx, const uint8_t* const* left1, const uint8_t* const* right1, size_t pitch, int channels);
VO_API int vo_mseq_submit_sized(vo_ctx* ctx, const uint8_t* const* left1, const uint8_t* const* right1,
                                const size_t* pitch, int channels);
/* Sequences that start while others run (a service whose streams come and go, or a queue of drives of unequal length).
 *   vo_mseq_open          ends a running sequence mode as vo_mseq_begin* do and opens a run of n_slots EMPTY slots whose
 *                         image planes, per-slot state, mono scratch (flag VO_MSEQ_MONO_ROTATION) and pinned block are
 *                         allocated once, at the envelope max_w x max_h.  An empty slot's wait status is VO_MSEQ_RETIRED
 *                         (zeroed record), its pose the identity, its state empty.
 *   vo_mseq_submit_start  vo_mseq_submit_sized plus n_start starts: starts[i].slot's pair of this call is the FIRST pair of
 *                         a new sequence of size w x h with the matrices P_l / P_r.  The slot may be empty, retired, or
 *                         live (its sequence then ends at its previous frame).  This submission only stages the pair and
 *                         builds its pyramids, as vo_seq_begin does; its wait reports VO_MSEQ_STARTED with a zeroed record
 *                         (and mono), and from that wait on the slot's pose is the identity and its state empty.  Waits
 *                         for earlier submissions still report the slot's previous sequence.  From the next submission
 *                         on the slot's pairs are plain pairs (a NULL pair retires it).  vo_mseq_submit_sized is this call
 *                         with n_start = 0.
 * A started sequence gives what vo_seq_begin(first pair) + vo_seq_push with its matrices gives on a fresh context, bit for
 * bit, and every other sequence what it gives without the start.  A start costs no kernel launch, and never allocates,
 * drains or synchronises; the front graph is recaptured only for a larger bucket grid than the run has seen.  Starts work
 * in runs of vo_mseq_begin* too (vo_mseq_begin / _ex / _calib runs: at the run's one size only).
 * Refused, changing nothing: VO_E_INVALID for a slot out of range, two starts in one slot, a start without both images,
 * pitch[slot] < channels * w, w or h <= 0, a third submission in flight, and vo_mseq_open with n_slots outside
 * 1 .. VO_MSEQ_MAX or while the other sequence mode has frames in flight or a batch submission has not been waited for;
 * VO_E_UNSUPPORTED for a size outside the envelope, of another pyramid depth, with h / 10 == 0, or other than the one size
 * of a run begun with one size; VO_E_CAPACITY for a size whose bucket grid exceeds the bucketing scratch (4096 cells) or,
 * with VO_MSEQ_MONO_ROTATION, the mono scratch (sized for the bucket grid of the envelope, or of the begun sizes). */
#define VO_MSEQ_STARTED 3        /* vo_mseq_wait status: this submission started the slot's sequence from its first pair */
typedef struct vo_mseq_start {
    int slot;                /* 0 <= slot < n_seq; the first pair is left1[slot] / right1[slot] of the same call */
    int w, h;                /* the new sequence's image size */
    float P_l[12], P_r[12];  /* its matrices, row-major 3 x 4, built as the reference's main() builds them (src/main.cpp:67-74) */
} vo_mseq_start;
VO_API int vo_mseq_open(vo_ctx* ctx, int n_slots, int max_w, int max_h, int flags);
VO_API int vo_mseq_submit_start(vo_ctx* ctx, const uint8_t* const* left1, const uint8_t* const* right1, const size_t* pitch,
                                int channels, int n_start, const vo_mseq_start* starts);
/* Frames already in device memory (vo_dimage, see vo_seq_begin_device), one descriptor pair per sequence.  Stream contract
 * as for the *_device calls above: the images are read after the work already enqueued on the context's stream, and work
 * the caller enqueues there after the call returns is ordered after the library's last read of them.  Each image has its
 * own format, pitch, strides and alignment (gray, BGR / RGB interleaved or planar), so the sequences of one call may
 * differ in layout; sequence q's images are read as its own w x h (its begun size, or its start's size).
 *   vo_mseq_begin_device   vo_mseq_begin_sized with left0[q] / right0[q] in place of host pointers, pitches and channels:
 *                          sequence q is w[q] x h[q] with the matrices P_l + 12 q / P_r + 12 q; flags takes
 *                          VO_MSEQ_MONO_ROTATION.  Synchronous, as vo_seq_begin_device: when it returns the first pairs
 *                          have been read.
 *   vo_mseq_submit_device  vo_mseq_submit_start with left1[q] / right1[q] in place of host pointers, pitches and channels
 *                          (n_start = 0: a plain submission).  A pair whose two data pointers are NULL retires its
 *                          sequence, as a NULL host pair does.  Results through vo_mseq_wait[_mono], vo_mseq_pose and
 *                          vo_mseq_state.
 * Both work in every multi-sequence run (begun with any vo_mseq_begin*, with vo_mseq_begin_device or with vo_mseq_open),
 * and host and device submissions may alternate within a run.  Each sequence's results are those of the same pixels (as
 * cv::cvtColor(BGR2GRAY / RGB2GRAY) converts colour) through the host entry points, bit for bit.  The 2 * n_seq images of a
 * submission are converted by ONE kernel launch on the sequence mode's copy stream under the frame in flight, outside the
 * front stage's graph, so a device submission costs one launch more than a host gray submission whatever n_seq is; each
 * image is checked with one cudaPointerGetAttributes.  Refused with VO_E_INVALID, changing nothing: NULL left / right
 * tables, an image that vo_seq_begin_device refuses (at its sequence's width), one NULL image in a pair, a pair for a
 * retired sequence, and every refusal of vo_mseq_begin_sized / vo_mseq_submit_start (with their codes). */
VO_API int vo_mseq_begin_device(vo_ctx* ctx, int n_seq, const int* w, const int* h, const float* P_l, const float* P_r,
                                const vo_dimage* left0, const vo_dimage* right0, int flags);
VO_API int vo_mseq_submit_device(vo_ctx* ctx, const vo_dimage* left1, const vo_dimage* right1, int n_start,
                                 const vo_mseq_start* starts);
VO_API int vo_mseq_wait(vo_ctx* ctx, vo_unit_result* out, int* status, vo_point2f* pts4, int pts_cap);
VO_API int vo_mseq_wait_mono(vo_ctx* ctx, vo_unit_result* out, int* status, vo_mono_result* mono,
                             uint8_t* ess_mask, int mask_cap, vo_point2f* pts4, int pts_cap);
/* Results into GPU memory, without a host wait: a device-resident loop (frames in from GPU memory, results out to it, the
 * host never touching pixels or waiting for a pose solve).  A run begun with the flag VO_MSEQ_DEVICE_RESULTS (any
 * vo_mseq_begin*, vo_mseq_begin_device or vo_mseq_open; it combines with VO_MSEQ_MONO_ROTATION):
 *   - takes its frames through vo_mseq_submit_device only, starts included (a begin with host pairs is synchronous and
 *     accepted).  Host submissions are refused: a wait that does not block gives no point after which a pinned host image
 *     is free again.
 *   - returns its results through vo_mseq_wait_device only; vo_mseq_wait / vo_mseq_wait_mono are refused.
 *   - keeps frame_pose on the device; vo_mseq_pose returns it after the last waited submission (it synchronises, as
 *     vo_mseq_state does).
 *   vo_mseq_wait_device  retires the oldest submission without blocking the host: ONE kernel launch on the context's
 *                        stream, ordered after the work already enqueued there and after that submission's pose solve
 *                        (never behind the next submission's), writes for every sequence q into the caller's device
 *                        buffers below; work enqueued on the context's stream after the call sees the results.  Every
 *                        pointer may be NULL (skipped); each must otherwise be device (or managed) memory of the context's
 *                        GPU.  The point arrays hold pts_cap entries per sequence, of which the first n_valid (inliers:
 *                        n_inliers) are defined; a retired or started sequence defines none.
 *     status[q]      VO_OK, VO_E_CAPACITY (glue error bits, as vo_mseq_wait; no message, the call returns VO_OK),
 *                    VO_MSEQ_RETIRED or VO_MSEQ_STARTED
 *     records[q]     vo_mseq_wait's record (zeroed for a retired or started slot)
 *     frame_pose     [n_seq][16] row-major: integrated in wait order under the main loop's gates, bit for bit as
 *                    vo_pose_step integrates it in vo_mseq_wait (the identity from a start on)
 *     pts4           [n_seq][4][pts_cap]: L0, R0, L1, R1, as vo_mseq_wait's pts4
 *     points3d       [n_seq][pts_cap]: points3D_t0, the triangulated L0 / R0 (vo_triangulate with the sequence's matrices)
 *     inliers        [n_seq][pts_cap]: solvePnPRansac's inliers, indices into the frame's n_valid list (vo_batch_outputs)
 *     mono, ess_mask [n_seq], [n_seq][pts_cap]: vo_mseq_wait_mono's, in runs with VO_MSEQ_MONO_ROTATION only
 *   Refused with VO_E_INVALID, changing nothing: a run without the flag, nothing in flight, pts_cap < 0, a point array
 *   with pts_cap == 0, mono / ess_mask without VO_MSEQ_MONO_ROTATION, a pointer that is not device memory of the
 *   context's GPU.  At most two submissions in flight, as ever. */
#define VO_MSEQ_DEVICE_RESULTS 8 /* vo_mseq_begin* / vo_mseq_open flag: results through vo_mseq_wait_device (bits 2 and 4 stay unknown) */
typedef struct vo_mseq_dresults {
    int32_t* status;             /* [n_seq] */
    vo_unit_result* records;     /* [n_seq] */
    double* frame_pose;          /* [n_seq][16] */
    int pts_cap;                 /* entries per sequence of pts4 (per list), points3d, inliers, ess_mask */
    vo_point2f* pts4;            /* [n_seq][4][pts_cap] */
    vo_point3f* points3d;        /* [n_seq][pts_cap] */
    int32_t* inliers;            /* [n_seq][pts_cap] */
    vo_mono_result* mono;        /* [n_seq] */
    uint8_t* ess_mask;           /* [n_seq][pts_cap] */
} vo_mseq_dresults;
VO_API int vo_mseq_wait_device(vo_ctx* ctx, const vo_mseq_dresults* r);
VO_API int vo_mseq_pose(vo_ctx* ctx, int q, double frame_pose[16]);
VO_API int vo_mseq_state(vo_ctx* ctx, int q, vo_point2f* points, int32_t* ages, int cap, int* n_points, int* n_ages, double t_out[3]);

/* ---- image ingest (SURVEY.md 8f, row N3) ---------------------------------------------------------------
 * What loadImageLeft / loadImageRight do (reference src/utils.cpp:172-190): read <dir>/image_0/%06d.png and
 * <dir>/image_1/%06d.png with cv::imread(IMREAD_COLOR) and cvtColor(BGR2GRAY).  The decoder is host code
 * (zlib inflate is a serial stream); the reader decodes AHEAD of the consumer on worker threads into a ring of
 * pinned buffers, so vo_seq_push's upload is one async DMA per image.
 *   vo_png_info / vo_png_decode   one PNG held in memory -> BGR (3 B/px) and/or gray (1 B/px); either may be NULL.
 *                                 Non-interlaced PNGs of every colour type / bit depth; 16-bit -> 8-bit by the high
 *                                 byte, alpha dropped (what IMREAD_COLOR does).  Errors: vo_png_last_error().
 *   vo_reader_open                sequence_dir/image_{0,1}/%06d.png, frames first_frame .. first_frame+n_frames-1,
 *                                 `threads` decoders, `depth` (>= 3) frames of pinned ring.  force_channels: 0 = gray
 *                                 files are delivered as gray, colour files as BGR (device conversion); 1 / 3 force.
 *   vo_reader_next                blocks until the next frame is decoded; the returned pointers stay valid until the
 *                                 SECOND following vo_reader_next (so a frame handed to vo_seq_submit may still be
 *                                 uploading while the next one is requested) or vo_reader_close.
 *   vo_bgr_to_gray                the device conversion on host buffers (stage-level entry point, for parity tests) */
typedef struct vo_reader vo_reader;
VO_API int vo_png_info(const uint8_t* file_bytes, size_t n, int* w, int* h, int* color_type, int* bit_depth);
VO_API int vo_png_decode(const uint8_t* file_bytes, size_t n, uint8_t* bgr, size_t bgr_pitch, uint8_t* gray, size_t gray_pitch);
VO_API const char* vo_png_last_error(void);
VO_API vo_reader* vo_reader_open(const char* sequence_dir, int first_frame, int n_frames, int threads, int depth, int force_channels);
VO_API int vo_reader_next(vo_reader* rd, const uint8_t** left, const uint8_t** right, int* w, int* h, size_t* pitch,
                          int* channels, int* frame_id);
VO_API const char* vo_reader_error(vo_reader* rd);
VO_API void vo_reader_close(vo_reader* rd);
VO_API int vo_bgr_to_gray(vo_ctx* ctx, const uint8_t* bgr, size_t pitch, int w, int h, uint8_t* gray, size_t gray_pitch);

/* ---- pose bookkeeping (SURVEY.md 8f, row N2) -- host-only, O(1) per frame ---------------------------
 * R is row-major 3x3, t is 3x1, frame_pose / rigid_inv are row-major 4x4 (the reference's CV_64F Mats).
 *   vo_pose_is_rotation  replaces isRotationMatrix            (src/utils.cpp:93-102):  |I - R^T R|_F < 1e-6
 *   vo_pose_euler        replaces rotationMatrixToEulerAngles (src/utils.cpp:107-131): float x,y,z
 *   vo_pose_integrate    replaces integrateOdometryStereo     (src/utils.cpp:57-91):   rigid_inv (optional) =
 *                        [R|t;0 0 0 1]^-1; frame_pose *= rigid_inv iff 0.05 < |t| < 10.  Returns 1 when the
 *                        pose was advanced, 0 when the frame was skipped, <0 on a singular transform.
 *   vo_pose_step         the main loop's gate + integration    (src/main.cpp:196-208):  all |euler| < 0.1
 *   vo_seq_pose          frame_pose accumulated by vo_seq_push since vo_seq_begin
 *   vo_pose_step_device  vo_pose_step of n frames (frame_pose[16 i], R[9 i], t[3 i]; rc[i] its return value, rc may be
 *                        NULL) computed by the device function vo_mseq_wait_device integrates with (stage-level entry
 *                        point, for parity tests; synchronous) */
VO_API int  vo_pose_is_rotation(const double R[9]);
VO_API void vo_pose_euler(const double R[9], float euler_xyz[3]);
VO_API int  vo_pose_integrate(double frame_pose[16], const double R[9], const double t[3], double rigid_inv[16]);
VO_API int  vo_pose_step(double frame_pose[16], const double R[9], const double t[3]);
VO_API int  vo_seq_pose(vo_ctx* ctx, double frame_pose[16]);
VO_API int  vo_pose_step_device(vo_ctx* ctx, int n, double* frame_pose, const double* R, const double* t, int* rc);

/* ---- KITTI accuracy evaluation (SURVEY.md 8f, row N4) -- host-only, offline -----------------------------
 * Poses are KITTI rows: 12 doubles = top 3 rows of the 4x4 camera-to-world matrix (what vo_seq_pose accumulates).
 *   vo_poses_load / vo_poses_save   replace loadPoses (src/evaluate/evaluate_odometry.cpp:17-33; also read by
 *                                   src/main.cpp for the ground-truth overlay) and the result writer
 *   vo_eval_segments                replaces calcSequenceErrors (evaluate_odometry.cpp:71-116): start every `step`
 *                                   (10) frames, segment lengths `lengths` (NULL = 100..800 m) along the ground-truth
 *                                   path; per segment r_err [rad/m], t_err [fraction], speed [m/s at 10 Hz]
 *   vo_eval_summary                 replaces saveStats (evaluate_odometry.cpp:376-395): mean t_err, r_err
 * With out == NULL vo_eval_segments / vo_poses_load only count. */
typedef struct vo_segment_error { int32_t first_frame; float r_err, t_err, len, speed; } vo_segment_error;
VO_API int vo_poses_load(const char* path, double* poses12, int cap, int* n_out);
VO_API int vo_poses_save(const char* path, const double* poses12, int n);
VO_API int vo_eval_segments(const double* gt12, const double* est12, int n_poses, const float* lengths, int n_lengths,
                            int step, vo_segment_error* out, int cap, int* n_out);
VO_API int vo_eval_summary(const vo_segment_error* seg, int n, float* t_err_avg, float* r_err_avg);

#ifdef __cplusplus
}
#endif
#endif /* VO_B200_H */
