// batch.cu -- the batched, device-resident whole-path API (vo_batch_*, vo_frame_batch).
//
// One call runs, for every resident work unit and with no host round trip in between:
//   [FAST on L0 + even-stride selection]  ->  pyramids  ->  LK ring (L0->R0->R1->L1->L0)
//   ->  status / negative-coordinate / circular filters  ->  DLT triangulation  ->  PnP/RANSAC + LM
// i.e. reference src/visualOdometry.cpp:81-129 (matchingFeatures, with the bucketing replaced by
// the benchmark's stride selection), src/main.cpp:170-171 and src/visualOdometry.cpp:132-193.
#include "ctx.h"
#include <string.h>
#include <algorithm>
#include <type_traits>

__global__ void k_pack_counts(vo_unit_result_dev* res, const int* n_pts, const int* n_det, const int* n3, const int* n5,
                              int n_units, int detect)
{
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_units) return;
    res[u].n_features = n_pts[u];
    res[u].n_detected = detect ? n_det[u] : 0;
    res[u].n_tracked = n3[u];
    res[u].n_valid = n5[u];
}

// Packed outputs of one unit: float2 pts4[4][per] (L0, R0, L1, R1 of the valid tracks) | int kept_idx[per] |
// float3 X[per] | int inliers[per] [| uint8 ess_mask[per]], `per` point slots each (only the first n_valid / n_inliers are
// written).  The mask section exists once a unit of the context ran the mono_rotation branch (ctx->out_mask); it is
// written for the units whose switch on[u] is set, from their five-point scratch blocks mask_stride bytes apart.
#define VO_OUT_BYTES_PER_SLOT (4 * sizeof(float2) + sizeof(int) + sizeof(float3) + sizeof(int))
__global__ void k_pack_outputs(uint8_t* __restrict__ out, size_t stride, int per, const float2* __restrict__ valid4, size_t cs,
                               const int* __restrict__ idx5, const float3* __restrict__ X, const int* __restrict__ inliers,
                               const int* __restrict__ n5, const vo_unit_result_dev* __restrict__ res, int cap,
                               const uint8_t* __restrict__ mask, size_t mask_stride, const int* __restrict__ on)
{
    const int u = blockIdx.x;
    const int nv = min(n5[u], per), ni = min(res[u].n_inliers, per);
    float2* o4 = reinterpret_cast<float2*>(out + (size_t)u * stride);
    int* ok = reinterpret_cast<int*>(o4 + 4 * (size_t)per);
    float* oX = reinterpret_cast<float*>(ok + per);
    int* oi = reinterpret_cast<int*>(oX + 3 * (size_t)per);
    const size_t ub = (size_t)u * cap;
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
#pragma unroll
        for (int k = 0; k < 4; k++) o4[(size_t)k * per + i] = valid4[k * cs + ub + i];
        ok[i] = idx5[ub + i];
        const float3 x = X[ub + i];
        oX[3 * i] = x.x; oX[3 * i + 1] = x.y; oX[3 * i + 2] = x.z;
    }
    for (int i = threadIdx.x; i < ni; i += blockDim.x) oi[i] = inliers[ub + i];
    if (mask && on[u]) {
        uint8_t* om = reinterpret_cast<uint8_t*>(oi + per);
        for (int i = threadIdx.x; i < nv; i += blockDim.x) om[i] = mask[(size_t)u * mask_stride + i];
    }
}

// the point count of each unit's mono_rotation problem: its n_valid when its switch is on, else 0 (no RANSAC work)
__global__ void k_batch_mono_n(int* __restrict__ n_out, const int* __restrict__ on, const int* __restrict__ n5, int n_units)
{
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u < n_units) n_out[u] = on[u] ? n5[u] : 0;
}

// the four parts of one unit's packed block with `per` point slots (layout of k_pack_outputs)
struct PackedUnit { float2* o4; int* ok; float* oX; int* oi; uint8_t* om; };
static PackedUnit packed_unit(uint8_t* base, int per)
{
    PackedUnit p;
    p.o4 = (float2*)base;
    p.ok = (int*)(p.o4 + 4 * (size_t)per);
    p.oX = (float*)(p.ok + per);
    p.oi = (int*)(p.oX + 3 * (size_t)per);
    p.om = (uint8_t*)(p.oi + per);
    return p;
}

// whether a unit of [u0, u0 + n) has the mono_rotation branch switched on
static bool range_mono(const vo_ctx* ctx, int u0, int n)
{
    for (int u = u0; u < u0 + n && u < (int)ctx->batch_mono.size(); u++)
        if (ctx->batch_mono[u]) return true;
    return false;
}

// largest feature bound of the slots [u0, u0 + n): the LK launch of that range has no unit with more live features
static int range_bound(const vo_ctx* ctx, int u0, int n)
{
    int b = 0;
    for (int u = u0; u < u0 + n && u < (int)ctx->slot_pts.size(); u++) b = ctx->slot_pts[u] > b ? ctx->slot_pts[u] : b;
    return b;
}

// Device + pinned blocks of the packed outputs before a submission of slots [u0, u0 + n) whose units carry at most
// `bound` features.  `per` is the largest bound over the resident slots, so it never drops below what a submission that
// is still in flight, or waited for but not yet read, has packed.  On a resize those submissions are completed first
// (they stay pending for vo_batch_wait) and every unit's lists are moved into the new layout.
static int ensure_outputs(vo_ctx* ctx, int u0, int n, int bound)
{
    int per = bound;
    for (int u = 0; u < (int)ctx->slot_pts.size(); u++)
        if ((u < u0 || u >= u0 + n) && ctx->slot_pts[u] > per) per = ctx->slot_pts[u];
    per = ((per > 1 ? per : 1) + 63) / 64 * 64;
    if (per > ctx->cap) per = ctx->cap;
    const bool mask = ctx->batch_mono_used;
    if (ctx->d_out && ctx->h_out && ctx->out_per == per && ctx->out_mask == mask && ctx->out_units >= ctx->units) return VO_OK;
    const size_t stride = ((size_t)per * (VO_OUT_BYTES_PER_SLOT + (mask ? 1 : 0)) + 255) / 256 * 256;
    for (auto& p : ctx->pending)                // their copies land in the old blocks
        if (p.active) VO_CUDA_CHECK(cudaEventSynchronize(p.done));
    int rc = vo_sync_device_retired(ctx);       // so do those of device-waited submissions still running
    if (rc) return rc;
    void* q = nullptr;                         // both new blocks first: a failed allocation leaves the old ones in use
    VO_CUDA_CHECK(cudaMalloc(&q, stride * ctx->units + 256));
    uint8_t* h = nullptr;
    const cudaError_t e = cudaMallocHost(&h, stride * ctx->units + 256);
    if (e != cudaSuccess) { cudaFree(q); VO_CUDA_CHECK(e); }
    if (ctx->h_out) {
        const int nu = ctx->out_units < ctx->units ? ctx->out_units : ctx->units;
        const int m = ctx->out_per < per ? ctx->out_per : per;
        for (int u = 0; u < nu; u++) {
            const PackedUnit a = packed_unit(ctx->h_out + (size_t)u * ctx->out_stride, ctx->out_per), b = packed_unit(h + (size_t)u * stride, per);
            for (int k = 0; k < 4; k++) memcpy(b.o4 + (size_t)k * per, a.o4 + (size_t)k * ctx->out_per, (size_t)m * sizeof(float2));
            memcpy(b.ok, a.ok, (size_t)m * sizeof(int));
            memcpy(b.oX, a.oX, (size_t)m * 3 * sizeof(float));
            memcpy(b.oi, a.oi, (size_t)m * sizeof(int));
            if (mask && ctx->out_mask) memcpy(b.om, a.om, (size_t)m);
        }
        cudaFreeHost(ctx->h_out);
    }
    ctx->h_out = h;
    if (ctx->d_out) {                           // only a staging area for the D2H copies: nothing in it is kept
        ctx->allocs.erase(std::find(ctx->allocs.begin(), ctx->allocs.end(), (void*)ctx->d_out));
        cudaFree(ctx->d_out);
    }
    ctx->allocs.push_back(q);                   // freed with the batch state
    ctx->d_out = (uint8_t*)q;
    ctx->out_units = ctx->units; ctx->out_per = per; ctx->out_stride = stride; ctx->out_mask = mask;
    return VO_OK;
}

extern "C" int vo_batch_configure(vo_ctx* ctx, int w, int h, int n_units, const float P_l[12], const float P_r[12])
{
    if (!ctx) return VO_E_INVALID;
    if (!P_l || !P_r || n_units <= 0) { vo_set_error(ctx, "bad argument"); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    int rc = vo_claim_buffers(ctx, "vo_batch_configure");
    if (rc) return rc;
    if ((rc = vo_ensure_state(ctx, w, h, n_units))) return rc;
    if ((rc = vo_set_calibration(ctx, 0, ctx->units, P_l, P_r, 1))) return rc;        // every unit, as the resident state holds them
    const std::vector<UnitParams> e(ctx->units, vo_unit_params(ctx->p));              // and the context's parameters
    if ((rc = vo_write_params(ctx, 0, ctx->units, e.data()))) return rc;
    ctx->batch_units = n_units;
    ctx->batch_uploaded = 0;
    ctx->slot_pts.assign(n_units, 0);
    ctx->batch_mono.assign(n_units, 0);         // every unit off (the device switch table is rewritten when one is set)
    ctx->batch_mono_ran.assign(n_units, 0);
    ctx->batch_mono_used = false;
    return VO_OK;
}

// Refused while submissions are in flight (they read the table); an idle sequence is ended, as by vo_batch_configure,
// since its units may be among those set.  The write is queued on the context's stream, ahead of every later submission.
extern "C" int vo_batch_calibrate(vo_ctx* ctx, int first_unit, int n_units, const float* P_l, const float* P_r)
{
    if (!ctx) return VO_E_INVALID;
    if (!P_l || !P_r) { vo_set_error(ctx, "vo_batch_calibrate: null projection matrices"); return VO_E_INVALID; }
    if (first_unit < 0 || n_units <= 0 || first_unit + n_units > ctx->batch_units) {
        vo_set_error(ctx, "vo_batch_calibrate: units [%d, %d) outside the configured batch (%d)", first_unit, first_unit + n_units, ctx->batch_units);
        return VO_E_INVALID;
    }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    int rc = vo_claim_buffers(ctx, "vo_batch_calibrate");
    if (rc) return rc;
    return vo_set_calibration(ctx, first_unit, n_units, P_l, P_r, n_units);
}

// the same rules as vo_batch_calibrate; each entry checked before anything changes
extern "C" int vo_batch_params(vo_ctx* ctx, int first_unit, int n_units, const vo_params* p)
{
    if (!ctx) return VO_E_INVALID;
    if (first_unit < 0 || n_units <= 0 || first_unit + n_units > ctx->batch_units) {
        vo_set_error(ctx, "vo_batch_params: units [%d, %d) outside the configured batch (%d)", first_unit, first_unit + n_units, ctx->batch_units);
        return VO_E_INVALID;
    }
    int rc;
    std::vector<UnitParams> e(n_units, vo_unit_params(ctx->p));
    for (int i = 0; p && i < n_units; i++) {
        char what[32];
        snprintf(what, sizeof(what), "unit %d", first_unit + i);
        if ((rc = vo_check_unit_params(ctx, "vo_batch_params", what, p[i]))) return rc;
        e[i] = vo_unit_params(p[i]);
    }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    if ((rc = vo_claim_buffers(ctx, "vo_batch_params"))) return rc;
    return vo_write_params(ctx, first_unit, n_units, e.data());
}

// the same rules as vo_batch_calibrate.  The scratch (one block per configured unit) is allocated here, never by a
// submission; the whole switch table is then written on the context's stream, ahead of every later submission.
extern "C" int vo_batch_mono_rotation(vo_ctx* ctx, int first_unit, int n_units, const uint8_t* on)
{
    if (!ctx) return VO_E_INVALID;
    if (first_unit < 0 || n_units <= 0 || first_unit + n_units > ctx->batch_units) {
        vo_set_error(ctx, "vo_batch_mono_rotation: units [%d, %d) outside the configured batch (%d)", first_unit, first_unit + n_units, ctx->batch_units);
        return VO_E_INVALID;
    }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    int rc = vo_claim_buffers(ctx, "vo_batch_mono_rotation");
    if (rc) return rc;
    if ((rc = vo_ensure_unit_ess(ctx, ctx->batch_units))) return rc;
    if (ctx->batch_mono_cap < ctx->batch_units) {
        int* q = nullptr;
        VO_CUDA_CHECK(cudaMalloc(&q, 2 * (size_t)ctx->batch_units * sizeof(int)));
        vo_drop_graphs(ctx);                    // captured graphs hold the old table
        if (ctx->d_batch_mono) { VO_CUDA_CHECK(cudaDeviceSynchronize()); cudaFree(ctx->d_batch_mono); }
        ctx->d_batch_mono = q; ctx->batch_mono_cap = ctx->batch_units;
    }
    for (int i = 0; i < n_units; i++) ctx->batch_mono[first_unit + i] = on && on[i] ? 1 : 0;
    if (range_mono(ctx, 0, ctx->batch_units)) ctx->batch_mono_used = true;
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_batch_mono, ctx->batch_mono.data(), (size_t)ctx->batch_units * sizeof(int),
                                  cudaMemcpyHostToDevice, ctx->stream));
    return VO_OK;
}

// Pinned staging of the batched path, disjoint per unit: t_prev [batch_units][3] | counts [batch_units] | result records
// [batch_units] (64-byte aligned) | descriptors of caller device images [batch_units][4] | mono_rotation results
// [batch_units]
static size_t batch_pinned_bytes(const vo_ctx* ctx)
{
    return (size_t)ctx->batch_units * (3 * sizeof(double) + sizeof(int) + sizeof(vo_unit_result_dev) + 4 * sizeof(vo_dimage) +
                                       sizeof(EssResult)) + 256;
}

static vo_unit_result_dev* pinned_results(vo_ctx* ctx)
{
    char* p = (char*)ctx->h_pinned + (size_t)ctx->batch_units * (3 * sizeof(double) + sizeof(int));
    p = (char*)(((uintptr_t)p + 63) & ~(uintptr_t)63);
    return (vo_unit_result_dev*)p;
}

static vo_dimage* pinned_ingest_tab(vo_ctx* ctx) { return (vo_dimage*)(pinned_results(ctx) + ctx->batch_units); }

static EssResult* pinned_ess(vo_ctx* ctx) { return (EssResult*)(pinned_ingest_tab(ctx) + 4 * (size_t)ctx->batch_units); }

// features and scalars of units [u0, u0+n) on stream `st`, through the pinned staging block; units[src0 + i] fills slot u0 + i
template <typename Unit>
static int stage_inputs(vo_ctx* ctx, const Unit* units, int u0, int n, cudaStream_t st, bool detect, int src0)
{
    const int cap = ctx->cap;
    const int total = ctx->batch_units;
    double* h_tprev = (double*)ctx->h_pinned;
    int* h_cnt = (int*)(h_tprev + 3 * (size_t)total);
    for (int u = u0; u < u0 + n; u++) {
        const Unit& U = units[u - u0 + src0];
        if (!detect && U.n_pts > 0)
            VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_pts_in + (size_t)u * cap, U.pts, (size_t)U.n_pts * sizeof(float2),
                                          cudaMemcpyHostToDevice, st));
        h_cnt[u] = U.n_pts;
        ctx->slot_pts[u] = U.n_pts;
        for (int k = 0; k < 3; k++) h_tprev[3 * u + k] = U.t_prev[k];
    }
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_tprev + 3 * (size_t)u0, h_tprev + 3 * (size_t)u0, (size_t)n * 3 * sizeof(double),
                                  cudaMemcpyHostToDevice, st));
    VO_CUDA_CHECK(cudaMemcpyAsync((detect ? ctx->d_want : ctx->d_npts) + u0, h_cnt + u0, (size_t)n * sizeof(int),
                                  cudaMemcpyHostToDevice, st));
    return VO_OK;
}

// H2D of units [u0, u0+n) on stream `st`: the host images, then features and scalars
static int upload_range(vo_ctx* ctx, const vo_unit* units, int u0, int n, size_t pitch, cudaStream_t st, bool detect, int src0 = -1)
{
    if (src0 < 0) src0 = u0;           // units[src0 + i] fills resident slot u0 + i
    const int w = ctx->w, h = ctx->h;
    for (int u = u0; u < u0 + n; u++) {
        const vo_unit& U = units[u - u0 + src0];
        const uint8_t* imgs[4] = {U.l0, U.r0, U.l1, U.r1};
        for (int k = 0; k < 4; k++) {
            const int rc = vo_upload_plane(ctx, ctx->d_raw + ((size_t)u * 4 + k) * w * h, imgs[k], w, h, pitch, st);
            if (rc) return rc;
        }
    }
    return stage_inputs(ctx, units, u0, n, st, detect, src0);
}

static int check_images(vo_ctx* ctx, const vo_unit& U, int u, size_t pitch)
{
    if (pitch < (size_t)ctx->w) { vo_set_error(ctx, "pitch %zu < width %d", pitch, ctx->w); return VO_E_INVALID; }
    if (!U.l0 || !U.r0 || !U.l1 || !U.r1) { vo_set_error(ctx, "unit %d: null image", u); return VO_E_INVALID; }
    return VO_OK;
}

static int check_images(vo_ctx* ctx, const vo_dunit& U, int u, size_t)
{
    char who[64];
    snprintf(who, sizeof(who), "vo_batch_submit_device: unit %d", u);
    const vo_dimage* imgs[4] = {&U.l0, &U.r0, &U.l1, &U.r1};
    static const char* names[4] = {"l0", "r0", "l1", "r1"};
    for (int k = 0; k < 4; k++) {
        const int rc = vo_check_dimage(ctx, who, names[k], imgs[k], ctx->w);
        if (rc) return rc;
    }
    return VO_OK;
}

template <typename Unit>
static int validate_units(vo_ctx* ctx, const Unit* units, int n_units, size_t pitch, bool* detect_out, int* max_pts_out = nullptr)
{
    if (!ctx || !units) return VO_E_INVALID;
    if (n_units <= 0 || n_units > ctx->batch_units) { vo_set_error(ctx, "n_units=%d outside the configured batch (%d)", n_units, ctx->batch_units); return VO_E_INVALID; }
    const bool detect = (units[0].pts == nullptr);
    int max_pts = 0;
    for (int u = 0; u < n_units; u++) {
        const Unit& U = units[u];
        int rc = check_images(ctx, U, u, pitch);
        if (rc) return rc;
        if ((U.pts == nullptr) != detect) { vo_set_error(ctx, "units must all carry features or all request detection"); return VO_E_INVALID; }
        if (U.n_pts < 0 || U.n_pts > ctx->cap) { vo_set_error(ctx, "unit %d: n_pts=%d outside [0,%d]", u, U.n_pts, ctx->cap); return VO_E_CAPACITY; }
        if (U.n_pts > max_pts) max_pts = U.n_pts;
    }
    *detect_out = detect;
    if (max_pts_out) *max_pts_out = max_pts;
    return vo_ensure_pinned(ctx, batch_pinned_bytes(ctx));
}

extern "C" int vo_batch_upload(vo_ctx* ctx, const vo_unit* units, int n_units, size_t pitch)
{
    bool detect;
    int rc = validate_units(ctx, units, n_units, pitch, &detect);
    if (rc) return rc;
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    if ((rc = vo_claim_buffers(ctx, "vo_batch_upload", true))) return rc;
    if ((rc = vo_drain_pending(ctx))) return rc;
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));      // staging block may still be in flight
    if ((rc = upload_range(ctx, units, 0, n_units, pitch, ctx->stream, detect))) return rc;
    ctx->batch_uploaded = n_units;
    ctx->batch_detect = detect;
    return VO_OK;
}

// high-priority helper streams: the short and the latency-bound kernels of a range (FAST, pyramids, filters,
// triangulation, PnP) are issued there, the LK ring at normal priority on the lane's side stream.  With two ranges in
// flight the helpers' few CTAs are then never queued behind the thousands of pending CTAs of the OTHER range's LK launch,
// so consecutive LK launches follow each other directly and the ramp-down of one (a feature-ring lasts ~0.3 ms) fills
// with the next.  The lanes' schedule when the SM partition is off (vo_partition_enable fills them in otherwise).
static int ensure_helpers(vo_ctx* ctx)
{
    if (ctx->lane[0].pre) return VO_OK;
    int lo = 0, hi = 0;
    VO_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));      // hi is the numerically smallest value
    for (auto& L : ctx->lane) {
        VO_CUDA_CHECK(cudaStreamCreateWithPriority(&L.pre, cudaStreamNonBlocking, hi));
        VO_CUDA_CHECK(cudaStreamCreateWithPriority(&L.mono, cudaStreamNonBlocking, hi));
        L.post = L.pre;
        L.lk = L.side;
    }
    return VO_OK;
}

// the whole path for the resident units of `v`, asynchronous on v.s.  A range on a lane's side stream runs the lane's
// schedule (ctx.h, vo_ctx::Lane); any other range runs on v.s alone.
static int run_range_launch(vo_ctx* ctx, const View& v)
{
    int rc;
    View pre = v, lk = v, post = v;              // FAST + pyramids / the LK ring / the kernels after the ring
    cudaEvent_t* ev = nullptr;
    // the five-point kernels of the mono_rotation branch, forked from post after the filters and joined before the fold
    cudaStream_t mono_s = ctx->mono_stream;
    cudaEvent_t mono_ev[2] = {ctx->mono_ev[0], ctx->mono_ev[1]};
    for (auto& L : ctx->lane)
        if (L.side && v.s == L.side) {
            if ((rc = ensure_helpers(ctx))) return rc;
            pre.s = L.pre; lk.s = L.lk; post.s = L.post; ev = L.ev;
            mono_s = L.mono; mono_ev[0] = L.ev[4]; mono_ev[1] = L.ev[5];
        }
    const bool mono = range_mono(ctx, v.u0, v.n);
    // work on `to` after the work enqueued so far on `from`
    auto hand_over = [&](int k, cudaStream_t from, cudaStream_t to) -> int {
        if (from == to) return VO_OK;
        VO_CUDA_CHECK(cudaEventRecord(ev[k], from));
        VO_CUDA_CHECK(cudaStreamWaitEvent(to, ev[k], 0));
        return VO_OK;
    };
    if ((rc = hand_over(0, v.s, pre.s))) return rc;
    if (ctx->batch_detect) {
        if ((rc = vo_run_fast(ctx, pre, 0, false, ctx->d_par))) return rc;
        if ((rc = vo_run_select(ctx, pre))) return rc;
    }
    if ((rc = vo_run_pyramid(ctx, v.u0 * v.imgs, v.n * v.imgs, pre.s))) return rc;
    if ((rc = hand_over(1, pre.s, lk.s))) return rc;
    const int ip[4] = {0, 1, 3, 2}, in[4] = {1, 3, 2, 0};      // ring L0->R0->R1->L1->L0 (planes L0,R0,L1,R1)
    if ((rc = vo_run_lk_ring(ctx, lk, 4, ip, in, false, ctx->d_par))) return rc;
    if ((rc = hand_over(2, lk.s, post.s))) return rc;
    if ((rc = vo_run_filter(ctx, post, false, ctx->d_par))) return rc;
    EssArgs e;
    if (mono) {     // findEssentialMat + recoverPose on (L0, L1) of the units switched on, beside triangulation and PnP
        int* count = ctx->d_batch_mono + ctx->batch_mono_cap + v.u0;
        e = vo_unit_ess_args(ctx, v.u0, v.n, v.max_pts, count);
        VO_CUDA_CHECK(cudaEventRecord(mono_ev[0], post.s));
        VO_CUDA_CHECK(cudaStreamWaitEvent(mono_s, mono_ev[0], 0));
        k_batch_mono_n<<<(v.n + 63) / 64, 64, 0, mono_s>>>(count, ctx->d_batch_mono + v.u0, ctx->d_n5 + v.u0, v.n);
        ctx->launches += 1 + vo_launch_essential(e, mono_s);
        VO_CUDA_CHECK(cudaGetLastError());
        VO_CUDA_CHECK(cudaEventRecord(mono_ev[1], mono_s));
    }
    const size_t cs = (size_t)ctx->units * ctx->cap;
    if ((rc = vo_run_triangulate(ctx, post, ctx->d_valid4, ctx->d_valid4 + cs, ctx->d_n5, ctx->d_cal))) return rc;
    if ((rc = vo_run_pnp(ctx, post, ctx->d_valid4 + 2 * cs, ctx->d_n5, ctx->d_cal, ctx->d_par))) return rc;
    k_pack_counts<<<(v.n + 63) / 64, 64, 0, post.s>>>(ctx->d_results + v.u0, ctx->d_npts + v.u0, ctx->d_ndet + v.u0, ctx->d_n3 + v.u0,
                                                     ctx->d_n5 + v.u0, v.n, ctx->batch_detect ? 1 : 0);
    ctx->launches += 1;
    if (mono) {     // the record's R becomes recoverPose's rotation (I where the branch aborted) for the units switched on
        VO_CUDA_CHECK(cudaStreamWaitEvent(post.s, mono_ev[1], 0));
        ctx->launches += vo_launch_mono_fold(ctx->d_results + v.u0, e.result, e.result_stride, ctx->d_batch_mono + v.u0, v.n, post.s);
    }
    VO_CUDA_CHECK(cudaGetLastError());
    return hand_over(3, post.s, v.s);            // join: later work on v.s (result copy, the next submission) sees everything
}

// The kernel sequence of the units [u0, u0 + n) on `s`.  On ctx->stream it is replayed (or first captured) as a CUDA
// graph: all kernel arguments are device pointers / sizes fixed by (range, feature bound, detect, staging), so the graph
// is reusable until the device state is re-allocated.  A range on a side stream is launched plainly: its kernels fork to
// the lane's partition or high-priority streams, which kernel nodes of a captured graph do not keep, and that split is
// worth more (+7 % on the pipelined step) than the graph's launch savings (+2 %).
static int run_range(vo_ctx* ctx, int u0, int n, cudaStream_t s)
{
    View v{u0, n, s};
    v.max_pts = range_bound(ctx, u0, n);         // the LK launch geometry depends on it
    for (int u = u0; u < u0 + n; u++) ctx->batch_mono_ran[u] = ctx->batch_mono[u];
    bool on_side = false;
    for (const auto& L : ctx->lane) on_side = on_side || (L.side && s == L.side);
    if (on_side) return run_range_launch(ctx, v);
    GraphKey key{};
    key.kind = GraphKey::BATCH_RANGE; key.s = s;
    key.u0 = u0; key.n = n; key.max_pts = v.max_pts; key.detect = ctx->batch_detect; key.mono = range_mono(ctx, u0, n);
    return vo_run_graph(ctx, key, [&] { return run_range_launch(ctx, v); });
}

extern "C" int vo_batch_run(vo_ctx* ctx)
{
    if (!ctx) return VO_E_INVALID;
    const int units = ctx->batch_uploaded;
    if (units <= 0) { vo_set_error(ctx, "vo_batch_run: nothing uploaded"); return VO_E_INVALID; }
    { int rcc = vo_claim_buffers(ctx, "vo_batch_run"); if (rcc) return rcc; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    if (units < 2 || ctx->batch_streams < 2) return run_range(ctx, 0, units, ctx->stream);
    // two unit ranges on two side streams: the latency-bound PnP kernels of one range run under the
    // LK ring of the other (fork from / join into the context's stream, so callers see one stream)
    int rc = vo_ensure_lanes(ctx);
    if (rc) return rc;
    VO_CUDA_CHECK(cudaEventRecord(ctx->fork_ev, ctx->stream));
    const int half = (units + 1) / 2;
    for (int c = 0; c < 2; c++) {
        const int u0 = c ? half : 0, n = c ? units - half : half;
        cudaStream_t st = ctx->lane[c].side;
        VO_CUDA_CHECK(cudaStreamWaitEvent(st, ctx->fork_ev, 0));
        if ((rc = run_range(ctx, u0, n, st))) return rc;
        VO_CUDA_CHECK(cudaEventRecord(ctx->lane[c].join, st));
        VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->lane[c].join, 0));
    }
    return VO_OK;
}

extern "C" int vo_batch_download(vo_ctx* ctx, vo_unit_result* results, int n_units)
{
    if (!ctx || !results) return VO_E_INVALID;
    if (n_units <= 0 || n_units > ctx->batch_uploaded) { vo_set_error(ctx, "n_units=%d outside the resident batch (%d)", n_units, ctx->batch_uploaded); return VO_E_INVALID; }
    static_assert(sizeof(vo_unit_result) == sizeof(vo_unit_result_dev), "result record layout");
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    VO_CUDA_CHECK(cudaMemcpyAsync(results, ctx->d_results, (size_t)n_units * sizeof(vo_unit_result), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}

// End-to-end entry point: H2D + whole path + D2H.  The batch is split into two unit ranges on two
// side streams forked from / joined into the context's stream, so the H2D of the second range runs
// under the kernels of the first (the images arrive over PCIe; compute is ~6x longer than the copy).
extern "C" int vo_frame_batch(vo_ctx* ctx, const vo_unit* units, int n_units, size_t pitch, vo_unit_result* results)
{
    bool detect;
    int rc = validate_units(ctx, units, n_units, pitch, &detect);
    if (rc) return rc;
    if (!results) return VO_E_INVALID;
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    if ((rc = vo_claim_buffers(ctx, "vo_frame_batch", true))) return rc;
    if ((rc = vo_drain_pending(ctx))) return rc;
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->batch_uploaded = n_units; ctx->batch_detect = detect;
    vo_unit_result_dev* h_res = pinned_results(ctx);
    const int nchunks = (n_units >= 2 && ctx->batch_streams >= 2) ? 2 : 1;
    if (nchunks == 1) {
        if ((rc = upload_range(ctx, units, 0, n_units, pitch, ctx->stream, detect))) return rc;
        if ((rc = run_range(ctx, 0, n_units, ctx->stream))) return rc;
        VO_CUDA_CHECK(cudaMemcpyAsync(h_res, ctx->d_results, (size_t)n_units * sizeof(vo_unit_result_dev), cudaMemcpyDeviceToHost, ctx->stream));
    } else {
        if ((rc = vo_ensure_lanes(ctx))) return rc;
        VO_CUDA_CHECK(cudaEventRecord(ctx->fork_ev, ctx->stream));
        const int half = (n_units + 1) / 2;
        for (int c = 0; c < 2; c++) {
            const int u0 = c ? half : 0, n = c ? n_units - half : half;
            cudaStream_t st = ctx->lane[c].side;
            VO_CUDA_CHECK(cudaStreamWaitEvent(st, ctx->fork_ev, 0));
            if ((rc = upload_range(ctx, units, u0, n, pitch, st, detect))) return rc;
            if ((rc = run_range(ctx, u0, n, st))) return rc;
            VO_CUDA_CHECK(cudaMemcpyAsync(h_res + u0, ctx->d_results + u0, (size_t)n * sizeof(vo_unit_result_dev), cudaMemcpyDeviceToHost, st));
            VO_CUDA_CHECK(cudaEventRecord(ctx->lane[c].join, st));
            VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->lane[c].join, 0));
        }
    }
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    memcpy(results, h_res, (size_t)n_units * sizeof(vo_unit_result));
    return VO_OK;
}

// ---- pipelined submissions -------------------------------------------------------------------------------------
// A submission fills the resident unit slots [first_unit, first_unit + n_units), runs the whole path on them and
// copies their result records to pinned staging, all asynchronously on one of the two side streams (alternating).
// Submissions on disjoint slot ranges overlap on the GPU: the H2D copy, FAST / pyramids and above all the
// latency-bound PnP tail (a few warps for ~0.4 ms) of one run under the issue-bound LK ring of the other, which a
// synchronous vo_frame_batch per batch cannot do for its last unit range.
//
// Host units: H2D copies of the images on the lane stream.  Device units (vo_batch_submit_device): one k_bgr_to_gray
// launch for the range on the lane stream, which follows fork_ev and so the caller's work on ctx->stream (producer
// ordering); ctx->stream then waits for that launch only, which releases the caller's images without waiting for the range.
static int upload_units(vo_ctx* ctx, const vo_unit* units, int u0, int n, size_t pitch, cudaStream_t st, int, bool detect)
{
    return upload_range(ctx, units, u0, n, pitch, st, detect, 0);
}

static int upload_units(vo_ctx* ctx, const vo_dunit* units, int u0, int n, size_t, cudaStream_t st, int lane, bool detect)
{
    vo_dimage* tab = pinned_ingest_tab(ctx) + 4 * (size_t)u0;
    for (int i = 0; i < n; i++) {
        tab[4 * i] = units[i].l0; tab[4 * i + 1] = units[i].r0; tab[4 * i + 2] = units[i].l1; tab[4 * i + 3] = units[i].r1;
    }
    int rc = vo_ingest_device(ctx, tab, 4 * n, 4 * u0, st);
    if (rc) return rc;
    VO_CUDA_CHECK(cudaEventRecord(ctx->lane[lane].join, st));
    VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->lane[lane].join, 0));
    return stage_inputs(ctx, units, u0, n, st, detect, 0);
}

template <typename Unit>
static int batch_submit(vo_ctx* ctx, const char* who, const Unit* units, int first_unit, int n_units, size_t pitch)
{
    if (!ctx) return VO_E_INVALID;
    if (first_unit < 0 || n_units <= 0 || first_unit + n_units > ctx->batch_units) {
        vo_set_error(ctx, "%s: slots [%d, %d) outside the configured batch (%d)", who, first_unit, first_unit + n_units, ctx->batch_units);
        return VO_E_INVALID;
    }
    { int rcc = vo_claim_buffers(ctx, who, true); if (rcc) return rcc; }
    for (auto& p : ctx->pending)
        if (p.active && first_unit < p.u0 + p.n && p.u0 < first_unit + n_units) {
            vo_set_error(ctx, "%s: slots [%d, %d) overlap a submission that has not been waited for", who, first_unit, first_unit + n_units);
            return VO_E_INVALID;
        }
    bool detect = ctx->batch_detect; int max_pts = 0;
    int rc;
    if (units) {
        if ((rc = validate_units(ctx, units, n_units, pitch, &detect, &max_pts))) return rc;
    } else {
        if (ctx->batch_uploaded < first_unit + n_units) {
            vo_set_error(ctx, "%s: units == NULL but slots [%d, %d) were never uploaded", who, first_unit, first_unit + n_units);
            return VO_E_INVALID;
        }
        if ((rc = vo_ensure_pinned(ctx, batch_pinned_bytes(ctx)))) return rc;
        max_pts = range_bound(ctx, first_unit, n_units);
    }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    if ((rc = vo_ensure_lanes(ctx))) return rc;
    if (ctx->part_auto) {
        // Pipelined submissions: the persistent LK ring of one range would keep the latency-bound kernels after the other
        // range's ring (filters, triangulation, PnP) off the SMs until it ends.  8 SMs are set aside for them (green
        // contexts); FAST / pyramids stay with the ring.  Measured: value 4239 -> 4603, e2e 3854 -> 4540 frames/s.
        ctx->part_auto = false;
        if (vo_partition_enable(ctx, 8) != VO_OK) ctx->err[0] = 0;      // no green contexts on this driver: run unpartitioned
    }
    if (ctx->batch_outputs && (rc = ensure_outputs(ctx, first_unit, n_units, max_pts))) return rc;
    // A device-waited submission of these units may not have copied its pinned staging to the device yet: the host
    // rewrites that staging below only after those copies (never after its pose solve).
    for (auto& p : ctx->pending)
        if (units && p.device_retired && first_unit < p.u0 + p.n && p.u0 < first_unit + n_units)
            VO_CUDA_CHECK(cudaEventSynchronize(p.staged));
    // a free record: neither in flight nor possibly still running after a device wait
    vo_ctx::Pending* slot = nullptr;
    for (auto& p : ctx->pending) {
        if (p.active) continue;
        if (p.device_retired) {
            const cudaError_t e = cudaEventQuery(p.done);
            if (e == cudaSuccess) p.device_retired = false;
            else if (e != cudaErrorNotReady) VO_CUDA_CHECK(e);
        }
        if (!p.device_retired) { slot = &p; break; }
    }
    if (!slot) {
        ctx->pending.emplace_back();
        slot = &ctx->pending.back();
        VO_CUDA_CHECK(cudaEventCreateWithFlags(&slot->done, cudaEventDisableTiming));
        VO_CUDA_CHECK(cudaEventCreateWithFlags(&slot->staged, cudaEventDisableTiming));
    }
    const int c = (int)((ctx->submit_count++) % VO_LANES);     // up to VO_LANES submissions in flight, each on its own lane
    cudaStream_t st = ctx->lane[c].side;
    // The lane follows everything on ctx->stream, including the k_seq_collect launch of a vo_batch_wait_device of these
    // slots: a range resubmitted right after a device wait overwrites its unit buffers only once they have been read.
    VO_CUDA_CHECK(cudaEventRecord(ctx->fork_ev, ctx->stream));
    VO_CUDA_CHECK(cudaStreamWaitEvent(st, ctx->fork_ev, 0));
    if ((rc = vo_dist_order_after_gathers(ctx, st))) return rc;
    ctx->batch_detect = detect;
    if (units) {
        if ((rc = upload_units(ctx, units, first_unit, n_units, pitch, st, c, detect))) return rc;
        if (ctx->batch_uploaded < first_unit + n_units) ctx->batch_uploaded = first_unit + n_units;
    }
    const bool device_in = !units || std::is_same<Unit, vo_dunit>::value;
    if (device_in) VO_CUDA_CHECK(cudaEventRecord(slot->staged, st));
    if ((rc = run_range(ctx, first_unit, n_units, st))) return rc;
    vo_unit_result_dev* h_res = pinned_results(ctx);
    VO_CUDA_CHECK(cudaMemcpyAsync(h_res + first_unit, ctx->d_results + first_unit, (size_t)n_units * sizeof(vo_unit_result_dev), cudaMemcpyDeviceToHost, st));
    const bool mono = range_mono(ctx, first_unit, n_units);
    // the branch's results for vo_batch_wait_mono
    if (mono && (rc = vo_copy_unit_ess(ctx, pinned_ess(ctx) + first_unit, first_unit, n_units, st))) return rc;
    if (ctx->batch_outputs) {                    // the point lists of the submission: one packed block, one copy
        const size_t cs = (size_t)ctx->units * ctx->cap, ub = (size_t)first_unit * ctx->cap;
        EssArgs e;
        if (mono) e = vo_unit_ess_args(ctx, first_unit, n_units, ctx->cap, nullptr);
        k_pack_outputs<<<n_units, 256, 0, st>>>(ctx->d_out + (size_t)first_unit * ctx->out_stride, ctx->out_stride, ctx->out_per,
                                               ctx->d_valid4 + ub, cs, ctx->d_idx5 + ub, ctx->d_X + ub, ctx->d_inliers + ub,
                                               ctx->d_n5 + first_unit, ctx->d_results + first_unit, ctx->cap,
                                               mono ? e.mask : nullptr, ctx->unit_ess_bytes, ctx->d_batch_mono + first_unit);
        ctx->launches += 1;
        VO_CUDA_CHECK(cudaGetLastError());
        VO_CUDA_CHECK(cudaMemcpyAsync(ctx->h_out + (size_t)first_unit * ctx->out_stride, ctx->d_out + (size_t)first_unit * ctx->out_stride,
                                      (size_t)n_units * ctx->out_stride, cudaMemcpyDeviceToHost, st));
    }
    VO_CUDA_CHECK(cudaEventRecord(slot->done, st));
    slot->u0 = first_unit; slot->n = n_units; slot->active = true; slot->device_in = device_in;
    return VO_OK;
}

extern "C" int vo_batch_submit(vo_ctx* ctx, const vo_unit* units, int first_unit, int n_units, size_t pitch)
{
    return batch_submit(ctx, "vo_batch_submit", units, first_unit, n_units, pitch);
}

extern "C" int vo_batch_submit_device(vo_ctx* ctx, const vo_dunit* units, int first_unit, int n_units)
{
    return batch_submit(ctx, "vo_batch_submit_device", units, first_unit, n_units, 0);
}

// vo_mono_result of a unit whose last run had the branch on (status as vo_seq_wait_mono reports it), zeroed otherwise
static vo_mono_result mono_result(const vo_ctx* ctx, int unit, const EssResult& ess)
{
    vo_mono_result m;
    memset(&m, 0, sizeof(m));
    return ctx->batch_mono_ran[unit] ? vo_mono_from_ess(ess) : m;
}

static int batch_wait(vo_ctx* ctx, const char* who, int first_unit, int n_units, vo_unit_result* results, vo_mono_result* mono)
{
    if (!ctx) return VO_E_INVALID;
    for (auto& p : ctx->pending)
        if (p.active && p.u0 == first_unit && p.n == n_units) {
            VO_CUDA_CHECK(cudaSetDevice(ctx->device));
            VO_CUDA_CHECK(cudaEventSynchronize(p.done));
            VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, p.done, 0));     // later work on the caller's stream sees the results
            p.active = false;
            if (results) memcpy(results, pinned_results(ctx) + first_unit, (size_t)n_units * sizeof(vo_unit_result));
            for (int i = 0; mono && i < n_units; i++) mono[i] = mono_result(ctx, first_unit + i, pinned_ess(ctx)[first_unit + i]);
            return VO_OK;
        }
    vo_set_error(ctx, "%s: no pending submission for slots [%d, %d)", who, first_unit, first_unit + n_units);
    return VO_E_INVALID;
}

extern "C" int vo_batch_wait(vo_ctx* ctx, int first_unit, int n_units, vo_unit_result* results)
{
    return batch_wait(ctx, "vo_batch_wait", first_unit, n_units, results, nullptr);
}

extern "C" int vo_batch_wait_mono(vo_ctx* ctx, int first_unit, int n_units, vo_unit_result* results, vo_mono_result* mono)
{
    if (ctx && !mono) { vo_set_error(ctx, "vo_batch_wait_mono: null mono"); return VO_E_INVALID; }
    return batch_wait(ctx, "vo_batch_wait_mono", first_unit, n_units, results, mono);
}

// whether a unit of [u0, u0 + n) ran the mono_rotation branch in its last run
static bool range_mono_ran(const vo_ctx* ctx, int u0, int n)
{
    for (int u = u0; u < u0 + n && u < (int)ctx->batch_mono_ran.size(); u++)
        if (ctx->batch_mono_ran[u]) return true;
    return false;
}

// vo_batch_wait_device: ONE k_seq_collect launch on ctx->stream, after the caller's work there and after the submission's
// `done`; the host only moves its bookkeeping on.  The records are those the submission folded on the device (the bytes
// vo_batch_wait copies out of pinned staging); the lists come straight from the unit buffers, which a resubmission of the
// range overwrites only after this launch (it forks from ctx->stream).  The switch table d_batch_mono holds the switches
// the submission ran with: vo_batch_mono_rotation is refused while it is pending and queues its write behind this launch.
extern "C" int vo_batch_wait_device(vo_ctx* ctx, int first_unit, int n_units, const vo_batch_dresults* r)
{
    static const char* who = "vo_batch_wait_device";
    if (!ctx) return VO_E_INVALID;
    vo_ctx::Pending* p = nullptr;
    for (auto& q : ctx->pending)
        if (q.active && q.u0 == first_unit && q.n == n_units) { p = &q; break; }
    if (!p) {
        vo_set_error(ctx, "%s: no pending submission for slots [%d, %d)", who, first_unit, first_unit + n_units);
        return VO_E_INVALID;
    }
    if (!p->device_in) {
        vo_set_error(ctx, "%s: slots [%d, %d) were submitted from host images, which only vo_batch_wait releases", who,
                     first_unit, first_unit + n_units);
        return VO_E_INVALID;
    }
    if (!r) { vo_set_error(ctx, "%s: null result table", who); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const bool mono = range_mono_ran(ctx, first_unit, n_units);
    EssArgs e;
    if (mono) e = vo_unit_ess_args(ctx, first_unit, n_units, ctx->cap, nullptr);
    CollectArgs a;
    int rc;
    if ((rc = vo_collect_args(ctx, who, r, r->kept_idx != nullptr, first_unit, mono ? &e : nullptr, a)) ||
        (rc = vo_check_dptr(ctx, who, "kept_idx", r->kept_idx)))
        return rc;
    a.all_ran = true;
    a.idx5 = ctx->d_idx5 + (size_t)first_unit * ctx->cap; a.kept_out = r->kept_idx;
    if (mono) a.ess_on = ctx->d_batch_mono + first_unit;
    VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, p->done, 0));
    ctx->launches += vo_launch_seq_collect(a, n_units, ctx->stream);
    VO_CUDA_CHECK(cudaGetLastError());
    p->active = false;
    p->device_retired = true;
    return VO_OK;
}

// After vo_batch_wait_device the host reads of a unit (pinned staging, or the unit buffers) first wait for its submission.
static int sync_device_retired_unit(vo_ctx* ctx, int unit)
{
    for (auto& p : ctx->pending)
        if (p.device_retired && unit >= p.u0 && unit < p.u0 + p.n) {
            VO_CUDA_CHECK(cudaSetDevice(ctx->device));
            VO_CUDA_CHECK(cudaEventSynchronize(p.done));
            p.device_retired = false;
        }
    return VO_OK;
}

// VO_E_INVALID + message unless `unit` is resident and not part of a submission that has not been waited for
static int check_waited(vo_ctx* ctx, const char* who, int unit)
{
    if (unit < 0 || unit >= ctx->batch_uploaded) { vo_set_error(ctx, "%s: unit %d outside the resident batch", who, unit); return VO_E_INVALID; }
    for (auto& p : ctx->pending)
        if (p.active && unit >= p.u0 && unit < p.u0 + p.n) { vo_set_error(ctx, "%s: unit %d has not been waited for", who, unit); return VO_E_INVALID; }
    return sync_device_retired_unit(ctx, unit);
}

// The branch's result of the unit's last run and its mask (n_valid bytes, aligned with vo_batch_fetch's lists), read
// synchronously from the unit's scratch block.  A unit that ran with the branch off: mono zeroed, ess_mask untouched.
extern "C" int vo_batch_fetch_mono(vo_ctx* ctx, int unit, vo_mono_result* mono, uint8_t* ess_mask)
{
    if (!ctx) return VO_E_INVALID;
    if (!mono) { vo_set_error(ctx, "vo_batch_fetch_mono: null mono"); return VO_E_INVALID; }
    int rc = check_waited(ctx, "vo_batch_fetch_mono", unit);
    if (rc) return rc;
    EssResult ess;
    memset(&ess, 0, sizeof(ess));
    if (!ctx->batch_mono_ran[unit]) { *mono = mono_result(ctx, unit, ess); return VO_OK; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const EssArgs e = vo_unit_ess_args(ctx, unit, 1, ctx->cap, nullptr);
    vo_unit_result_dev r;
    VO_CUDA_CHECK(cudaMemcpyAsync(&r, ctx->d_results + unit, sizeof(r), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(&ess, e.result, sizeof(ess), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (ess_mask && r.n_valid > 0) {
        VO_CUDA_CHECK(cudaMemcpyAsync(ess_mask, e.mask, (size_t)std::min(r.n_valid, ctx->cap), cudaMemcpyDeviceToHost, ctx->stream));
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    }
    *mono = mono_result(ctx, unit, ess);
    return VO_OK;
}

// The point lists of a waited submission, from the pinned block its single D2H copy filled ("batch_outputs" = 1):
// pts4 = [4][n_valid] (L0, R0, L1, R1), kept_idx / X = [n_valid], inliers = [n_inliers]; counts are in the unit's record.
extern "C" int vo_batch_outputs(vo_ctx* ctx, int unit, vo_point2f* pts4, int32_t* kept_idx, vo_point3f* X, int32_t* inliers,
                                size_t* d2h_bytes_per_unit)
{
    if (!ctx) return VO_E_INVALID;
    if (!ctx->batch_outputs || !ctx->h_out) { vo_set_error(ctx, "vo_batch_outputs: option batch_outputs is off"); return VO_E_INVALID; }
    if (unit < 0 || unit >= ctx->batch_uploaded || unit >= ctx->out_units) { vo_set_error(ctx, "unit %d outside the resident batch", unit); return VO_E_INVALID; }
    for (auto& p : ctx->pending)
        if (p.active && unit >= p.u0 && unit < p.u0 + p.n) { vo_set_error(ctx, "vo_batch_outputs: unit %d has not been waited for", unit); return VO_E_INVALID; }
    int rc = sync_device_retired_unit(ctx, unit);
    if (rc) return rc;
    const vo_unit_result_dev& r = pinned_results(ctx)[unit];
    const int per = ctx->out_per;
    const int nv = r.n_valid < per ? r.n_valid : per, ni = r.n_inliers < per ? r.n_inliers : per;
    const PackedUnit o = packed_unit(ctx->h_out + (size_t)unit * ctx->out_stride, per);
    if (pts4) for (int k = 0; k < 4; k++) memcpy(pts4 + (size_t)k * nv, o.o4 + (size_t)k * per, (size_t)nv * sizeof(float2));
    if (kept_idx) memcpy(kept_idx, o.ok, (size_t)nv * sizeof(int));
    if (X) memcpy(X, o.oX, (size_t)nv * 3 * sizeof(float));
    if (inliers) memcpy(inliers, o.oi, (size_t)ni * sizeof(int));
    if (d2h_bytes_per_unit) *d2h_bytes_per_unit = ctx->out_stride;
    return VO_OK;
}

// vo_batch_outputs' counterpart for the branch: the result staged by the submission and the mask its packed copy carried
extern "C" int vo_batch_outputs_mono(vo_ctx* ctx, int unit, vo_mono_result* mono, uint8_t* ess_mask)
{
    if (!ctx) return VO_E_INVALID;
    if (!mono) { vo_set_error(ctx, "vo_batch_outputs_mono: null mono"); return VO_E_INVALID; }
    if (!ctx->batch_outputs || !ctx->h_out) { vo_set_error(ctx, "vo_batch_outputs_mono: option batch_outputs is off"); return VO_E_INVALID; }
    if (unit >= ctx->out_units) { vo_set_error(ctx, "vo_batch_outputs_mono: unit %d outside the resident batch", unit); return VO_E_INVALID; }
    int rc = check_waited(ctx, "vo_batch_outputs_mono", unit);
    if (rc) return rc;
    *mono = mono_result(ctx, unit, pinned_ess(ctx)[unit]);
    if (ess_mask && ctx->batch_mono_ran[unit] && ctx->out_mask) {
        const int per = ctx->out_per, nv = std::min(pinned_results(ctx)[unit].n_valid, per);
        if (nv > 0) memcpy(ess_mask, packed_unit(ctx->h_out + (size_t)unit * ctx->out_stride, per).om, (size_t)nv);
    }
    return VO_OK;
}

extern "C" int vo_batch_fetch(vo_ctx* ctx, int unit, vo_point2f* pts_in, vo_point2f* pts4, int32_t* kept_idx,
                              vo_point3f* X, int32_t* inliers)
{
    if (!ctx) return VO_E_INVALID;
    if (unit < 0 || unit >= ctx->batch_uploaded) { vo_set_error(ctx, "unit %d outside the resident batch", unit); return VO_E_INVALID; }
    int rc = sync_device_retired_unit(ctx, unit);
    if (rc) return rc;
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    vo_unit_result_dev r;
    VO_CUDA_CHECK(cudaMemcpyAsync(&r, ctx->d_results + unit, sizeof(r), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    const size_t cs = (size_t)ctx->units * ctx->cap, ub = (size_t)unit * ctx->cap;
    if (pts_in && r.n_features > 0)
        VO_CUDA_CHECK(cudaMemcpyAsync(pts_in, ctx->d_pts_in + ub, (size_t)r.n_features * sizeof(float2), cudaMemcpyDeviceToHost, ctx->stream));
    if (pts4 && r.n_valid > 0)
        for (int k = 0; k < 4; k++)
            VO_CUDA_CHECK(cudaMemcpyAsync(pts4 + (size_t)k * r.n_valid, ctx->d_valid4 + k * cs + ub, (size_t)r.n_valid * sizeof(float2),
                                          cudaMemcpyDeviceToHost, ctx->stream));
    if (kept_idx && r.n_valid > 0)
        VO_CUDA_CHECK(cudaMemcpyAsync(kept_idx, ctx->d_idx5 + ub, (size_t)r.n_valid * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (X && r.n_valid > 0)
        VO_CUDA_CHECK(cudaMemcpyAsync(X, ctx->d_X + ub, (size_t)r.n_valid * sizeof(float3), cudaMemcpyDeviceToHost, ctx->stream));
    if (inliers && r.n_inliers > 0)
        VO_CUDA_CHECK(cudaMemcpyAsync(inliers, ctx->d_inliers + ub, (size_t)r.n_inliers * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}
