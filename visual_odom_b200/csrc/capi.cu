// capi.cu -- extern "C" entry points with HOST buffers (the drop-in boundary, include/vo_b200.h).
#include "ctx.h"
#include <string.h>

static int upload_image(vo_ctx* ctx, int plane, const uint8_t* img, int w, int h, size_t pitch)
{
    return vo_upload_plane(ctx, ctx->d_raw + (size_t)plane * w * h, img, w, h, pitch, ctx->stream);
}

static int check_common(vo_ctx* ctx, int w, int h, size_t pitch, int n)
{
    if (!ctx) return VO_E_INVALID;
    if (w <= 0 || h <= 0 || pitch < (size_t)w) { vo_set_error(ctx, "bad image geometry %dx%d pitch %zu", w, h, pitch); return VO_E_INVALID; }
    if (n < 0) { vo_set_error(ctx, "negative point count"); return VO_E_INVALID; }
    if (n > ctx->cap) { vo_set_error(ctx, "n=%d exceeds context capacity max_features=%d", n, ctx->cap); return VO_E_CAPACITY; }
    return VO_OK;
}

extern "C" int vo_lk_track(vo_ctx* ctx, const uint8_t* prev, const uint8_t* next, int w, int h, size_t pitch,
                           const vo_point2f* prev_pts, int n, vo_point2f* next_pts, uint8_t* status, float* err)
{
    int rc = check_common(ctx, w, h, pitch, n);
    if (rc) return rc;
    if ((rc = vo_claim_buffers(ctx, "vo_lk_track"))) return rc;
    if (n == 0) return VO_OK;          // OpenCV's LK returns early on 0 points
    if (!prev || !next || !prev_pts || !next_pts || !status) { vo_set_error(ctx, "null argument"); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    rc = vo_ensure_state(ctx, w, h, 1);
    if (rc) return rc;
    if ((rc = upload_image(ctx, 0, prev, w, h, pitch))) return rc;
    if ((rc = upload_image(ctx, 1, next, w, h, pitch))) return rc;
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_pts_in, prev_pts, (size_t)n * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_npts, &n, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    const int ip[1] = {0}, in[1] = {1};
    if ((rc = vo_run_lk(ctx, View{0, 1, ctx->stream, -1, 2, n}, 1, ip, in, err != nullptr, ctx->d_par_tab))) return rc;
    VO_CUDA_CHECK(cudaMemcpyAsync(next_pts, ctx->d_pts_out, (size_t)n * sizeof(float2), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(status, ctx->d_status, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    if (err) VO_CUDA_CHECK(cudaMemcpyAsync(err, ctx->d_err, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}

extern "C" int vo_circular_match(vo_ctx* ctx, const uint8_t* l0, const uint8_t* r0, const uint8_t* l1,
                                 const uint8_t* r1, int w, int h, size_t pitch, const vo_point2f* pts_l0, int n,
                                 int32_t* ages_io, vo_point2f* o_l0, vo_point2f* o_r0, vo_point2f* o_l1,
                                 vo_point2f* o_r1, vo_point2f* o_l0_ret, uint8_t* status4, vo_point2f* raw4,
                                 int32_t* kept_idx, int* n_kept)
{
    int rc = check_common(ctx, w, h, pitch, n);
    if (rc) return rc;
    if ((rc = vo_claim_buffers(ctx, "vo_circular_match"))) return rc;
    if (n_kept) *n_kept = 0;
    if (n == 0) return VO_OK;
    if (!l0 || !r0 || !l1 || !r1 || !pts_l0) { vo_set_error(ctx, "null argument"); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    rc = vo_ensure_state(ctx, w, h, 1);
    if (rc) return rc;
    const uint8_t* imgs[4] = {l0, r0, l1, r1};
    for (int i = 0; i < 4; i++)
        if ((rc = upload_image(ctx, i, imgs[i], w, h, pitch))) return rc;
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_pts_in, pts_l0, (size_t)n * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_npts, &n, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    if (ages_io)
        VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_ages_in, ages_io, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    // ring order: L0->R0, R0->R1, R1->L1, L1->L0   (planes: L0=0, R0=1, L1=2, R1=3)
    const int ip[4] = {0, 1, 3, 2}, in[4] = {1, 3, 2, 0};
    if ((rc = vo_run_lk(ctx, View{0, 1, ctx->stream, -1, 4, n}, 4, ip, in, false, ctx->d_par_tab))) return rc;
    if ((rc = vo_run_filter(ctx, View{0, 1, ctx->stream}, ages_io != nullptr, ctx->d_par_tab))) return rc;
    int n3 = 0;
    VO_CUDA_CHECK(cudaMemcpyAsync(&n3, ctx->d_n3, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    const size_t cs = (size_t)ctx->units * ctx->cap;
    if (status4)
        for (int c = 0; c < 4; c++)
            VO_CUDA_CHECK(cudaMemcpyAsync(status4 + (size_t)c * n, ctx->d_status + c * cs, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    if (raw4)
        for (int c = 0; c < 4; c++)
            VO_CUDA_CHECK(cudaMemcpyAsync(raw4 + (size_t)c * n, ctx->d_pts_out + c * cs, (size_t)n * sizeof(float2), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));   // n3 is needed to size the remaining copies
    vo_point2f* outs[5] = {o_l0, o_r0, o_l1, o_r1, o_l0_ret};
    for (int k = 0; k < 5; k++)
        if (outs[k] && n3 > 0)
            VO_CUDA_CHECK(cudaMemcpyAsync(outs[k], ctx->d_kept5 + k * cs, (size_t)n3 * sizeof(float2), cudaMemcpyDeviceToHost, ctx->stream));
    if (kept_idx && n3 > 0)
        VO_CUDA_CHECK(cudaMemcpyAsync(kept_idx, ctx->d_idx3, (size_t)n3 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (ages_io && n3 > 0)
        VO_CUDA_CHECK(cudaMemcpyAsync(ages_io, ctx->d_ages_out, (size_t)n3 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (n_kept) *n_kept = n3;
    return VO_OK;
}

// ---------------------------------------------------------------------------------------------
static int ensure_any_state(vo_ctx* ctx)
{
    if (ctx->units > 0) return VO_OK;
    return vo_ensure_state(ctx, 64, 64, 1);
}

extern "C" int vo_fast_detect(vo_ctx* ctx, const uint8_t* img, int w, int h, size_t pitch, vo_point2f* out,
                              float* response, int cap, int* n_out)
{
    int rc = check_common(ctx, w, h, pitch, 0);
    if (rc) return rc;
    if ((rc = vo_claim_buffers(ctx, "vo_fast_detect"))) return rc;
    if (!img || !n_out || (cap > 0 && !out)) { vo_set_error(ctx, "null argument"); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    if ((rc = vo_ensure_state(ctx, w, h, 1))) return rc;
    if ((rc = upload_image(ctx, 0, img, w, h, pitch))) return rc;
    if ((rc = vo_run_fast(ctx, View{0, 1, ctx->stream}, 0, response != nullptr, ctx->d_par_tab))) return rc;
    int n = 0;
    VO_CUDA_CHECK(cudaMemcpyAsync(&n, ctx->d_ndet, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    *n_out = n;
    int m = n < cap ? n : cap;
    if (m > ctx->corner_cap) m = ctx->corner_cap;
    if (m > 0) {
        VO_CUDA_CHECK(cudaMemcpyAsync(out, ctx->d_corners, (size_t)m * sizeof(float2), cudaMemcpyDeviceToHost, ctx->stream));
        if (response) VO_CUDA_CHECK(cudaMemcpyAsync(response, ctx->d_resp, (size_t)m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    }
    if (n > m) { vo_set_error(ctx, "%d corners found, %d returned (capacity)", n, m); return VO_E_CAPACITY; }
    return VO_OK;
}

static int triangulate_impl(vo_ctx* ctx, const float P_l[12], const float P_r[12], const vo_point2f* pts_l,
                            const vo_point2f* pts_r, int n, vo_point3f* X, float* X4)
{
    if (!ctx) return VO_E_INVALID;
    if (n < 0 || !P_l || !P_r) { vo_set_error(ctx, "bad argument"); return VO_E_INVALID; }
    if (n == 0) return VO_OK;
    if (n > ctx->cap) { vo_set_error(ctx, "n=%d exceeds max_features=%d", n, ctx->cap); return VO_E_CAPACITY; }
    if (!pts_l || !pts_r || (!X && !X4)) { vo_set_error(ctx, "null argument"); return VO_E_INVALID; }
    { int rcc = vo_claim_buffers(ctx, "vo_triangulate"); if (rcc) return rcc; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    int rc = ensure_any_state(ctx);
    if (rc) return rc;
    CamCalib c = ctx->cal[0];           // the stage calls' entry: the sequence and batched units keep their cameras
    for (int k = 0; k < 12; k++) { c.Pl[k] = (double)P_l[k]; c.Pr[k] = (double)P_r[k]; }
    if ((rc = vo_write_calib(ctx, -1, 1, &c))) return rc;
    const size_t cs = (size_t)ctx->units * ctx->cap;
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_valid4, pts_l, (size_t)n * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_valid4 + cs, pts_r, (size_t)n * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_n5, &n, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    // the homogeneous points use the (then idle) A5 point lists 2..3 of unit 0 as scratch: n float4 = 2 n float2
    float4* d_X4 = X4 ? reinterpret_cast<float4*>(ctx->d_kept5) : nullptr;
    if ((rc = vo_run_triangulate(ctx, View{0, 1, ctx->stream}, ctx->d_valid4, ctx->d_valid4 + cs, ctx->d_n5, ctx->d_cal_tab, d_X4))) return rc;
    if (X) VO_CUDA_CHECK(cudaMemcpyAsync(X, ctx->d_X, (size_t)n * sizeof(float3), cudaMemcpyDeviceToHost, ctx->stream));
    if (X4) VO_CUDA_CHECK(cudaMemcpyAsync(X4, d_X4, (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}

extern "C" int vo_triangulate(vo_ctx* ctx, const float P_l[12], const float P_r[12], const vo_point2f* pts_l,
                              const vo_point2f* pts_r, int n, vo_point3f* X)
{
    return triangulate_impl(ctx, P_l, P_r, pts_l, pts_r, n, X, nullptr);
}

extern "C" int vo_triangulate_homogeneous(vo_ctx* ctx, const float P_l[12], const float P_r[12], const vo_point2f* pts_l,
                                          const vo_point2f* pts_r, int n, float* X4)
{
    return triangulate_impl(ctx, P_l, P_r, pts_l, pts_r, n, nullptr, X4);
}

extern "C" int vo_pnp_ransac(vo_ctx* ctx, const vo_point3f* X, const vo_point2f* x, int n, const float K[9],
                             double rvec_io[3], double tvec_io[3], int32_t* inliers, int* n_inliers,
                             double R_out[9], int* ransac_iters)
{
    if (!ctx) return VO_E_INVALID;
    if (n_inliers) *n_inliers = 0;
    if (n < 0 || !K || !rvec_io || !tvec_io) { vo_set_error(ctx, "bad argument"); return VO_E_INVALID; }
    if (n < 4) { vo_set_error(ctx, "solvePnPRansac needs >= 4 points (got %d); the reference aborts here", n); return VO_E_TOO_FEW_POINTS; }
    if (n > ctx->cap) { vo_set_error(ctx, "n=%d exceeds max_features=%d", n, ctx->cap); return VO_E_CAPACITY; }
    if (!X || !x) { vo_set_error(ctx, "null argument"); return VO_E_INVALID; }
    if (rvec_io[0] != 0 || rvec_io[1] != 0 || rvec_io[2] != 0) {
        vo_set_error(ctx, "non-zero initial rvec is not supported (the reference resets rvec to 0 every call, visualOdometry.cpp:162)");
        return VO_E_UNSUPPORTED;
    }
    { int rcc = vo_claim_buffers(ctx, "vo_pnp_ransac"); if (rcc) return rcc; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    int rc = ensure_any_state(ctx);
    if (rc) return rc;
    const size_t cs = (size_t)ctx->units * ctx->cap;
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_X, X, (size_t)n * sizeof(float3), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_valid4 + 2 * cs, x, (size_t)n * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_n5, &n, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_tprev, tvec_io, 3 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CamCalib c = ctx->cal[0];           // the stage calls' entry
    vo_calib_set_pnp(c, K);
    if ((rc = vo_write_calib(ctx, -1, 1, &c))) return rc;
    if ((rc = vo_run_pnp(ctx, View{0, 1, ctx->stream}, ctx->d_valid4 + 2 * cs, ctx->d_n5, ctx->d_cal_tab, ctx->d_par_tab))) return rc;
    vo_unit_result_dev r;
    VO_CUDA_CHECK(cudaMemcpyAsync(&r, ctx->d_results, sizeof(r), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 3; k++) { rvec_io[k] = r.rvec[k]; tvec_io[k] = r.tvec[k]; }
    if (R_out) for (int k = 0; k < 9; k++) R_out[k] = r.R[k];
    if (ransac_iters) *ransac_iters = r.ransac_iters;
    if (n_inliers) *n_inliers = r.n_inliers;
    if (inliers && r.n_inliers > 0) {
        VO_CUDA_CHECK(cudaMemcpyAsync(inliers, ctx->d_inliers, (size_t)r.n_inliers * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    }
    return VO_OK;
}

// ---- N5: the mono_rotation = true branch ---------------------------------------------------------------------------
extern "C" int vo_mono_rotation(vo_ctx* ctx, const vo_point2f* pts_t0, const vo_point2f* pts_t1, int n, double focal, double ppx,
                                double ppy, double R_out[9], uint8_t* mask_out, int* n_inliers, int* ransac_iters)
{
    if (!ctx) return VO_E_INVALID;
    if (n_inliers) *n_inliers = 0;
    if (n < 0 || !R_out || !(focal > 0)) { vo_set_error(ctx, "vo_mono_rotation: bad argument"); return VO_E_INVALID; }
    if (n < 5) { vo_set_error(ctx, "vo_mono_rotation: cv::findEssentialMat needs >= 5 points (got %d); the reference aborts here", n); return VO_E_TOO_FEW_POINTS; }
    if (!pts_t0 || !pts_t1) { vo_set_error(ctx, "null argument"); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const int iters = VO_ESS_ITERS;
    // one scratch block: points | count | camera | the kernels' scratch (vo_ess_bind).  Separate from the sequence mode's
    // per-frame scratch and calibration table, so this call never touches a sequence's state.
    auto up = [](size_t x) { return (x + 255) / 256 * 256; };
    const size_t o_p0 = 0, o_p1 = o_p0 + up((size_t)n * 8), o_n = o_p1 + up((size_t)n * 8), o_cal = o_n + up(sizeof(int)),
                 o_ess = o_cal + up(sizeof(CamCalib)), total = o_ess + vo_ess_scratch_bytes(n, iters);
    if (!ctx->d_ess || ctx->ess_cap < n) {
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_ess) { cudaFree(ctx->d_ess); ctx->d_ess = nullptr; }
        VO_CUDA_CHECK(cudaMalloc(&ctx->d_ess, total));
        ctx->ess_cap = n;
    }
    uint8_t* b = (uint8_t*)ctx->d_ess;
    EssArgs a;
    memset(&a, 0, sizeof(a));
    CamCalib cal;
    memset(&cal, 0, sizeof(cal));
    vo_calib_set_ess(cal, focal, ppx, ppy);
    vo_ess_bind(a, b + o_ess, n, iters);
    a.n = (const int*)(b + o_n);
    a.cal = (const CamCalib*)(b + o_cal);
    a.pts0 = (const float2*)(b + o_p0); a.pts1 = (const float2*)(b + o_p1);
    VO_CUDA_CHECK(cudaMemcpyAsync(b + o_cal, &cal, sizeof(cal), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(b + o_p0, pts_t0, (size_t)n * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(b + o_p1, pts_t1, (size_t)n * sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(b + o_n, &n, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    ctx->launches += vo_launch_essential(a, ctx->stream);
    VO_CUDA_CHECK(cudaGetLastError());
    EssResult r;
    VO_CUDA_CHECK(cudaMemcpyAsync(&r, a.result, sizeof(r), cudaMemcpyDeviceToHost, ctx->stream));
    if (mask_out) VO_CUDA_CHECK(cudaMemcpyAsync(mask_out, a.mask, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 9; k++) R_out[k] = r.R[k];
    if (n_inliers) *n_inliers = r.n_inliers;
    if (ransac_iters) *ransac_iters = r.iters;
    if (r.status == ESS_FIVE_CANDIDATES) {
        vo_set_error(ctx, "vo_mono_rotation: with exactly 5 points cv::findEssentialMat runs no RANSAC and returns all %d five-point "
                          "candidates stacked (%dx3); cv::recoverPose asserts E is 3x3, the reference aborts here", r.n_cand, 3 * r.n_cand);
        return VO_E_TOO_FEW_POINTS;
    }
    if (r.status != ESS_OK) { vo_set_error(ctx, "vo_mono_rotation: RANSAC found no essential matrix with more than 4 inliers (cv::recoverPose would fail on the empty E)"); return VO_E_TOO_FEW_POINTS; }
    return VO_OK;
}
