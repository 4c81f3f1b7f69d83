// ctx.cu -- context life-cycle, device state, TMA descriptor encoding, stage runners.
#include "ctx.h"
#include <string.h>
#include <stdlib.h>

void vo_set_error(vo_ctx* ctx, const char* fmt, ...)
{
    if (!ctx) return;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
    va_end(ap);
}

extern "C" void vo_default_params(vo_params* p)
{
    p->fast_threshold = 20;
    p->fast_nonmax = 1;
    p->lk_win = 21;
    p->lk_max_level = 3;
    p->lk_max_iters = 30;
    p->lk_epsilon = 0.01;
    p->lk_min_eig = 0.001;
    p->circ_threshold = 0;
    p->pnp_iterations = 500;
    p->pnp_reproj_error = 0.5f;
    p->pnp_confidence = (double)0.999f;   // the reference stores it in a float (visualOdometry.cpp:170)
    p->max_features = 8192;
    p->max_units = 1;
    p->refill_threshold = 2000;           // visualOdometry.cpp:95
    p->bucket_rows_divisor = 10;          // visualOdometry.cpp:106
    p->features_per_bucket = 1;           // visualOdometry.cpp:107
    p->bucket_age_threshold = 10;         // bucket.cpp:16
}

int vo_check_params(vo_ctx* ctx, const vo_params& p)
{
    if (p.fast_threshold < 0 || p.fast_threshold > 255) {
        // a pixel difference lies in [-255, 255]: other thresholds have no meaning (cv::FAST gives arbitrary lists for them)
        vo_set_error(ctx, "fast_threshold=%d outside [0,255]", p.fast_threshold);
        return VO_E_INVALID;
    }
    if (!(p.pnp_confidence > 0.0 && p.pnp_confidence < 1.0)) {
        // cv::solvePnPRansac asserts 0 < confidence < 1 (NaN included); outside it the iteration bound has no meaning
        vo_set_error(ctx, "pnp_confidence=%g outside (0,1)", p.pnp_confidence);
        return VO_E_INVALID;
    }
    if (p.bucket_rows_divisor <= 0) {
        vo_set_error(ctx, "bucket_rows_divisor=%d: bucket_size = rows / divisor needs a positive divisor", p.bucket_rows_divisor);
        return VO_E_INVALID;
    }
    if (p.features_per_bucket <= 0) {
        // Bucket::add_feature on a full bucket of max_size 0 reads ages[0] of an empty vector
        vo_set_error(ctx, "features_per_bucket=%d: a bucket holds at least one feature", p.features_per_bucket);
        return VO_E_INVALID;
    }
    if (p.lk_win < VO_WIN_MIN) {
        // cv::calcOpticalFlowPyrLK asserts winSize.width > 2 && winSize.height > 2
        vo_set_error(ctx, "lk_win=%d: the LK window must be at least %dx%d", p.lk_win, VO_WIN_MIN, VO_WIN_MIN);
        return VO_E_INVALID;
    }
    if (p.lk_win > VO_WIN_MAX) {
        vo_set_error(ctx, "lk_win=%d unsupported: the LK kernels are built for windows from %d to %d", p.lk_win, VO_WIN_MIN,
                     VO_WIN_MAX);
        return VO_E_UNSUPPORTED;
    }
    if (p.lk_max_level < 0 || p.lk_max_level >= VO_MAX_LEVELS) {
        vo_set_error(ctx, "lk_max_level=%d outside [0,%d]", p.lk_max_level, VO_MAX_LEVELS - 1);
        return VO_E_UNSUPPORTED;
    }
    return VO_OK;
}

int vo_check_unit_params(vo_ctx* ctx, const char* who, const char* what, const vo_params& p)
{
    int rc = vo_check_params(ctx, p);
    if (rc) {
        char msg[sizeof(ctx->err)];
        snprintf(msg, sizeof(msg), "%s", ctx->err);
        vo_set_error(ctx, "%s: %s: %s", who, what, msg);
        return rc;
    }
    // the pyramid depth, the window and the corner capacity are the context's
    const struct { const char* name; int v, c; } common[] = {
        {"lk_win", p.lk_win, ctx->p.lk_win}, {"lk_max_level", p.lk_max_level, ctx->p.lk_max_level},
        {"fast_nonmax", p.fast_nonmax, ctx->p.fast_nonmax}};
    for (const auto& f : common)
        if (f.v != f.c) {
            vo_set_error(ctx, "%s: %s: %s=%d differs from the context's %d (it is context-wide)", who, what, f.name, f.v, f.c);
            return VO_E_UNSUPPORTED;
        }
    // the RANSAC scratch holds the context's iteration count
    if (p.pnp_iterations > vo_pnp_iterations(ctx)) {
        vo_set_error(ctx, "%s: %s: pnp_iterations=%d above the context's %d (the RANSAC scratch is sized for it)", who, what,
                     p.pnp_iterations, vo_pnp_iterations(ctx));
        return VO_E_CAPACITY;
    }
    return VO_OK;
}

UnitParams vo_unit_params(const vo_params& p)
{
    UnitParams e;
    memset(&e, 0, sizeof(e));
    // calcOpticalFlowPyrLK clamps the criteria: maxCount to [0, 100], epsilon to [0, 10]
    e.max_iters = p.lk_max_iters < 0 ? 0 : p.lk_max_iters > 100 ? 100 : p.lk_max_iters;
    double eps = p.lk_epsilon;
    if (eps < 0.) eps = 0.; if (eps > 10.) eps = 10.;
    e.eps2 = eps * eps;
    e.min_eig = (float)p.lk_min_eig;
    const double thr = (double)p.pnp_reproj_error;      // float -> double, squared in double, stored float
    e.thr2 = (float)(thr * thr);
    e.confidence = p.pnp_confidence;
    e.pnp_iterations = p.pnp_iterations > 1 ? p.pnp_iterations : 1;   // cv::RANSACPointSetRegistrator runs at least one
    e.fast_threshold = p.fast_threshold;
    e.circ_threshold = p.circ_threshold;
    e.refill_threshold = p.refill_threshold;
    e.bucket_rows_divisor = p.bucket_rows_divisor;
    e.features_per_bucket = p.features_per_bucket;
    e.bucket_age_threshold = p.bucket_age_threshold;
    return e;
}

extern "C" int vo_create(int device, const vo_params* params, vo_ctx** out)
{
    if (!out) return VO_E_INVALID;
    *out = nullptr;
    vo_ctx* ctx = new vo_ctx();
    if (params) ctx->p = *params; else vo_default_params(&ctx->p);
    ctx->device = device;
    *out = ctx;      // returned even on failure so the caller can read vo_last_error()
    if (ctx->p.max_features <= 0) {
        vo_set_error(ctx, "max_features=%d: the per-unit feature capacity must be positive", ctx->p.max_features);
        return VO_E_INVALID;
    }
    int rc = vo_check_params(ctx, ctx->p);
    if (rc) return rc;
    ctx->slot_par.assign(VO_MSEQ_MAX, ctx->p);
    ctx->slot_rect_on.assign(VO_MSEQ_MAX, 0);
    ctx->slot_rect.assign(VO_MSEQ_MAX, vo_rectify{});
    ctx->d_rect.assign(VO_MSEQ_MAX, nullptr);
    ctx->rect_bytes.assign(VO_MSEQ_MAX, 0);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) {
        vo_set_error(ctx, "no CUDA device available (%s): this library has no CPU fallback", cudaGetErrorString(e));
        return VO_E_CUDA;
    }
    VO_CUDA_CHECK(cudaSetDevice(device));
    cudaDeviceProp prop;
    VO_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {      // sm_90a code runs on compute capability 9.0 and nothing else
        vo_set_error(ctx, "device %d is sm_%d%d; this library ships sm_90a code only", device, prop.major, prop.minor);
        return VO_E_UNSUPPORTED;
    }
    ctx->sm_count = prop.multiProcessorCount;
    VO_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    ctx->stream = ctx->own_stream;
    VO_CUDA_CHECK(vo_lk_prepare());
    ctx->cap = ctx->p.max_features;
    ctx->bucket_cap = 2 * (size_t)ctx->cap;
    VO_CUDA_CHECK(cudaMalloc(&ctx->d_lk_queue, LK_QUEUES * 2 * sizeof(int)));
    VO_CUDA_CHECK(cudaMemset(ctx->d_lk_queue, 0, LK_QUEUES * 2 * sizeof(int)));
    const char* sp = getenv("VO_LK_SPAN");          // force the LK work-item size (tests/test_gpu_lk_variants.py sets it per context with "lk_span")
    if (sp) ctx->lk_span = atoi(sp);
    return VO_OK;
}

extern "C" void vo_destroy(vo_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    vo_drain_pending(ctx);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    vo_dist_shutdown(ctx);
    vo_partition_destroy(ctx);
    vo_free_state(ctx);
    for (cudaEvent_t e : ctx->ev_pool) cudaEventDestroy(e);
    for (auto& p : ctx->pending) {
        if (p.done) cudaEventDestroy(p.done);
        if (p.staged) cudaEventDestroy(p.staged);
    }
    for (int k = 0; k < 2; k++) {
        if (ctx->seq_front_ev[k]) cudaEventDestroy(ctx->seq_front_ev[k]);
        if (ctx->seq_back_ev[k]) cudaEventDestroy(ctx->seq_back_ev[k]);
    }
    if (ctx->fork_ev) cudaEventDestroy(ctx->fork_ev);
    for (auto& L : ctx->lane) {
        if (L.join) cudaEventDestroy(L.join);
        if (L.side) cudaStreamDestroy(L.side);
        for (cudaEvent_t e : L.ev) if (e) cudaEventDestroy(e);
    }
    if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
    if (ctx->d_bgr) cudaFree(ctx->d_bgr);
    for (void* p : ctx->d_rect) if (p) cudaFree(p);
    for (void* p : ctx->rect_dead) cudaFree(p);
    if (ctx->d_rect_stage) cudaFree(ctx->d_rect_stage);
    if (ctx->d_lk_queue) cudaFree(ctx->d_lk_queue);
    if (ctx->d_ess) cudaFree(ctx->d_ess);
    if (ctx->d_unit_ess) cudaFree(ctx->d_unit_ess);
    if (ctx->d_batch_mono) cudaFree(ctx->d_batch_mono);
    for (cudaEvent_t e : ctx->mono_ev) if (e) cudaEventDestroy(e);
    if (ctx->mono_stream) cudaStreamDestroy(ctx->mono_stream);
    if (ctx->d_seq_pose) cudaFree(ctx->d_seq_pose);
    for (cudaEvent_t e : ctx->seq_tab_ev) if (e) cudaEventDestroy(e);
    if (ctx->h_out) cudaFreeHost(ctx->h_out);
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    delete ctx;
}

extern "C" const char* vo_last_error(const vo_ctx* ctx) { return ctx ? ctx->err : "null context"; }

extern "C" int vo_set_stream(vo_ctx* ctx, void* s)
{
    if (!ctx) return VO_E_INVALID;
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->stream = s ? (cudaStream_t)s : ctx->own_stream;
    return VO_OK;
}

extern "C" int vo_sync(vo_ctx* ctx)
{
    if (!ctx) return VO_E_INVALID;
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}

extern "C" int vo_set_option(vo_ctx* ctx, const char* key, double value)
{
    if (!ctx || !key) return VO_E_INVALID;
    if (strcmp(key, "batch_streams") == 0) { ctx->batch_streams = value >= 2 ? 2 : 1; return VO_OK; }
    if (strcmp(key, "batch_outputs") == 0) { ctx->batch_outputs = value >= 1; vo_drop_graphs(ctx); return VO_OK; }
    if (strcmp(key, "sm_partition") == 0) {          // k > 0: the kernels after the LK ring on k SMs of their own; 0: no partition
        if (value < 0) { vo_set_error(ctx, "sm_partition=%g: the number of SMs must not be negative", value); return VO_E_INVALID; }
        ctx->part_auto = false;
        return vo_partition_enable(ctx, (int)value);
    }
    if (strcmp(key, "lk_span") == 0) { ctx->lk_span = (int)value; vo_drop_graphs(ctx); return VO_OK; }
    if (strcmp(key, "graphs") == 0) { ctx->use_graphs = value >= 1; return VO_OK; }
    if (strcmp(key, "mono_rotation") == 0) { ctx->mono_opt = value >= 1; vo_drop_graphs(ctx); return VO_OK; }
    vo_set_error(ctx, "unknown option %s", key);
    return VO_E_INVALID;
}

extern "C" long long vo_kernel_launches(const vo_ctx* ctx) { return ctx ? ctx->launches : 0; }

extern "C" int vo_lk_kernel_time(vo_ctx* ctx, double* ms_total, long long* n, int reset)
{
    if (!ctx) return VO_E_INVALID;
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i + 1 < ctx->ev_used; i += 2) {
        float ms = 0.f;
        VO_CUDA_CHECK(cudaEventElapsedTime(&ms, ctx->ev_pool[i], ctx->ev_pool[i + 1]));
        ctx->lk_ms += ms;
        ctx->lk_n++;
    }
    ctx->ev_used = 0;
    if (ms_total) *ms_total = ctx->lk_ms;
    if (n) *n = ctx->lk_n;
    if (reset) { ctx->lk_ms = 0.0; ctx->lk_n = 0; }
    return VO_OK;
}

int vo_ensure_pinned(vo_ctx* ctx, size_t bytes)
{
    if (bytes <= ctx->h_pinned_bytes) return VO_OK;
    if (ctx->h_pinned) { cudaFreeHost(ctx->h_pinned); ctx->h_pinned = nullptr; ctx->h_pinned_bytes = 0; }
    VO_CUDA_CHECK(cudaMallocHost(&ctx->h_pinned, bytes));
    ctx->h_pinned_bytes = bytes;
    return VO_OK;
}

int vo_upload_plane(vo_ctx* ctx, uint8_t* dst, const uint8_t* src, size_t row_bytes, int h, size_t pitch, cudaStream_t st)
{
    if (pitch == row_bytes) VO_CUDA_CHECK(cudaMemcpyAsync(dst, src, row_bytes * h, cudaMemcpyHostToDevice, st));
    else VO_CUDA_CHECK(cudaMemcpy2DAsync(dst, row_bytes, src, pitch, row_bytes, h, cudaMemcpyHostToDevice, st));
    return VO_OK;
}

int vo_refuse_pending_batches(vo_ctx* ctx, const char* who)
{
    for (auto& p : ctx->pending)
        if (p.active) {
            vo_set_error(ctx, "%s: the vo_batch_submit submission of slots [%d, %d) has not been waited for", who, p.u0, p.u0 + p.n);
            return VO_E_INVALID;
        }
    return vo_sync_device_retired(ctx);
}

int vo_sync_device_retired(vo_ctx* ctx)
{
    for (auto& p : ctx->pending)
        if (p.device_retired) {
            VO_CUDA_CHECK(cudaEventSynchronize(p.done));
            p.device_retired = false;
        }
    return VO_OK;
}

int vo_claim_buffers(vo_ctx* ctx, const char* who, bool allow_pending_batches)
{
    if (ctx->seq_inflight > 0) {
        vo_set_error(ctx, "%s: %d frame(s) submitted with vo_seq_submit have not been waited for (this call would overwrite their buffers)", who, ctx->seq_inflight);
        return VO_E_INVALID;
    }
    int rc;
    if (!allow_pending_batches && (rc = vo_refuse_pending_batches(ctx, who))) return rc;
    ctx->seq_active = false;        // the sequence's image planes and per-frame buffers are reused from here on: vo_seq_begin again
    return VO_OK;
}

// ---------------------------------------------------------------------------------------------
// SM partition: two green contexts (CUDA driver API, resolved through the runtime so that the library does not link libcuda)
typedef CUresult (*PFN_cuDeviceGet)(CUdevice*, int);
typedef CUresult (*PFN_cuDeviceGetDevResource)(CUdevice, CUdevResource*, CUdevResourceType);
typedef CUresult (*PFN_cuDevSmResourceSplitByCount)(CUdevResource*, unsigned int*, const CUdevResource*, CUdevResource*, unsigned int, unsigned int);
typedef CUresult (*PFN_cuDevResourceGenerateDesc)(CUdevResourceDesc*, CUdevResource*, unsigned int);
typedef CUresult (*PFN_cuGreenCtxCreate)(CUgreenCtx*, CUdevResourceDesc, CUdevice, unsigned int);
typedef CUresult (*PFN_cuGreenCtxStreamCreate)(CUstream*, CUgreenCtx, unsigned int, int);
typedef CUresult (*PFN_cuGreenCtxDestroy)(CUgreenCtx);

template <typename F>
static bool drv(const char* name, F* fn)
{
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) return false;
    *fn = (F)p;
    return true;
}

// also drops the lanes' priority helpers: a lane without pre / lk / post streams gets them again on first use (batch.cu)
void vo_partition_destroy(vo_ctx* ctx)
{
    for (auto& L : ctx->lane) {
        if (L.pre) cudaStreamDestroy(L.pre);                            // partition: pre = lk; helpers: pre = post, lk = side
        if (L.post && L.post != L.pre) cudaStreamDestroy(L.post);
        if (L.mono) cudaStreamDestroy(L.mono);
        L.pre = L.lk = L.post = L.mono = nullptr;
    }
    PFN_cuGreenCtxDestroy destroy = nullptr;
    if (drv("cuGreenCtxDestroy", &destroy))
        for (int k = 0; k < 2; k++) if (ctx->part_gctx[k]) destroy((CUgreenCtx)ctx->part_gctx[k]);
    ctx->part_gctx[0] = ctx->part_gctx[1] = nullptr;
    ctx->part_on = false; ctx->part_helper_sms = ctx->part_lk_sms = 0;
}

int vo_partition_enable(vo_ctx* ctx, int helper_sms)
{
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    int rc = vo_drain_pending(ctx);
    if (rc) return rc;
    VO_CUDA_CHECK(cudaDeviceSynchronize());
    vo_drop_graphs(ctx);
    vo_partition_destroy(ctx);
    if (helper_sms <= 0) return VO_OK;
    PFN_cuDeviceGet dget; PFN_cuDeviceGetDevResource getres; PFN_cuDevSmResourceSplitByCount split;
    PFN_cuDevResourceGenerateDesc gendesc; PFN_cuGreenCtxCreate create; PFN_cuGreenCtxStreamCreate screate;
    if (!drv("cuDeviceGet", &dget) || !drv("cuDeviceGetDevResource", &getres) || !drv("cuDevSmResourceSplitByCount", &split) ||
        !drv("cuDevResourceGenerateDesc", &gendesc) || !drv("cuGreenCtxCreate", &create) || !drv("cuGreenCtxStreamCreate", &screate)) {
        vo_set_error(ctx, "sm_partition: this driver has no green-context API");
        return VO_E_UNSUPPORTED;
    }
    CUdevice dev;
    CUdevResource all, part[1], rest;
    unsigned int nb = 1;
    CUresult r;
    if ((r = dget(&dev, ctx->device)) != CUDA_SUCCESS || (r = getres(dev, &all, CU_DEV_RESOURCE_TYPE_SM)) != CUDA_SUCCESS ||
        (r = split(part, &nb, &all, &rest, 0, (unsigned)helper_sms)) != CUDA_SUCCESS || nb != 1) {
        vo_set_error(ctx, "sm_partition: splitting off %d SMs failed (driver error %d)", helper_sms, (int)r);
        return VO_E_UNSUPPORTED;
    }
    CUdevResource* rs[2] = {&part[0], &rest};
    for (int k = 0; k < 2; k++) {
        CUdevResourceDesc desc;
        CUgreenCtx g;
        if ((r = gendesc(&desc, rs[k], 1)) != CUDA_SUCCESS || (r = create(&g, desc, dev, CU_GREEN_CTX_DEFAULT_STREAM)) != CUDA_SUCCESS) {
            vo_set_error(ctx, "sm_partition: cuGreenCtxCreate failed (driver error %d)", (int)r);
            vo_partition_destroy(ctx);
            return VO_E_UNSUPPORTED;
        }
        ctx->part_gctx[k] = g;
    }
    ctx->part_helper_sms = (int)part[0].sm.smCount; ctx->part_lk_sms = (int)rest.sm.smCount;
    for (int c = 0; c < VO_LANES; c++) {
        CUstream a, b, m;
        if ((r = screate(&a, (CUgreenCtx)ctx->part_gctx[0], CU_STREAM_NON_BLOCKING, 0)) != CUDA_SUCCESS ||
            (r = screate(&b, (CUgreenCtx)ctx->part_gctx[1], CU_STREAM_NON_BLOCKING, 0)) != CUDA_SUCCESS ||
            (r = screate(&m, (CUgreenCtx)ctx->part_gctx[0], CU_STREAM_NON_BLOCKING, 0)) != CUDA_SUCCESS) {
            vo_set_error(ctx, "sm_partition: cuGreenCtxStreamCreate failed (driver error %d)", (int)r);
            vo_partition_destroy(ctx);
            return VO_E_UNSUPPORTED;
        }
        vo_ctx::Lane& L = ctx->lane[c];
        L.pre = L.lk = (cudaStream_t)b;
        L.post = (cudaStream_t)a;
        L.mono = (cudaStream_t)m;                                       // the five-point kernels beside post, on the same SMs
    }
    ctx->part_on = true;
    return VO_OK;
}

// wait for every vo_batch_submit that was not waited for (before state is re-allocated, re-used synchronously or freed)
int vo_drain_pending(vo_ctx* ctx)
{
    for (auto& p : ctx->pending)
        if (p.active) {
            VO_CUDA_CHECK(cudaEventSynchronize(p.done));
            p.active = false;
        }
    int rc = vo_sync_device_retired(ctx);
    if (rc) return rc;
    // frames of the sequence mode still in flight on the pose-solve stream
    if (ctx->seq_inflight > 0 && ctx->lane[0].side) VO_CUDA_CHECK(cudaStreamSynchronize(ctx->lane[0].side));
    return VO_OK;
}

// ---------------------------------------------------------------------------------------------
void vo_drop_graphs(vo_ctx* ctx)
{
    for (auto& g : ctx->graphs) cudaGraphExecDestroy(g.exec);
    ctx->graphs.clear();
}

static bool same_key(const GraphKey& a, const GraphKey& b)
{
    return a.kind == b.kind && a.s == b.s && a.u0 == b.u0 && a.n == b.n && a.max_pts == b.max_pts &&
           a.detect == b.detect && a.mono == b.mono && a.slot == b.slot && a.parity == b.parity && a.bgr == b.bgr;
}

int vo_run_graph(vo_ctx* ctx, const GraphKey& key, const std::function<int()>& launch)
{
    if (!ctx->use_graphs) return launch();
    for (auto& g : ctx->graphs)
        if (same_key(g.key, key)) {
            VO_CUDA_CHECK(cudaGraphLaunch(g.exec, key.s));
            ctx->launches += g.launches;
            return VO_OK;
        }
    const bool timing = ctx->lk_timing;
    const long long before = ctx->launches;
    ctx->lk_timing = false;
    cudaGraph_t graph = nullptr;
    VO_CUDA_CHECK(cudaStreamBeginCapture(key.s, cudaStreamCaptureModeThreadLocal));
    int rc = launch();
    cudaError_t e = cudaStreamEndCapture(key.s, &graph);
    ctx->lk_timing = timing;
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    VO_CUDA_CHECK(e);
    vo_ctx::CachedGraph g;
    g.key = key;
    g.launches = ctx->launches - before;
    VO_CUDA_CHECK(cudaGraphInstantiate(&g.exec, graph, 0));
    cudaGraphDestroy(graph);
    ctx->graphs.push_back(g);
    VO_CUDA_CHECK(cudaGraphLaunch(g.exec, key.s));
    return VO_OK;
}

int vo_ensure_lanes(vo_ctx* ctx)
{
    if (ctx->fork_ev) return VO_OK;
    VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->fork_ev, cudaEventDisableTiming));
    for (auto& L : ctx->lane) {
        VO_CUDA_CHECK(cudaStreamCreateWithFlags(&L.side, cudaStreamNonBlocking));
        VO_CUDA_CHECK(cudaEventCreateWithFlags(&L.join, cudaEventDisableTiming));
        for (cudaEvent_t& e : L.ev) VO_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    return VO_OK;
}

int vo_ensure_unit_ess(vo_ctx* ctx, int n_units)
{
    if (!ctx->mono_stream) {
        VO_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->mono_stream, cudaStreamNonBlocking));
        for (cudaEvent_t& e : ctx->mono_ev) VO_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    if (ctx->unit_ess_units >= n_units) return VO_OK;
    vo_drop_graphs(ctx);                                      // captured graphs hold the old blocks
    if (ctx->d_unit_ess) { VO_CUDA_CHECK(cudaDeviceSynchronize()); cudaFree(ctx->d_unit_ess); ctx->d_unit_ess = nullptr; ctx->unit_ess_units = 0; }
    const size_t bytes = (vo_ess_scratch_bytes(ctx->cap, VO_ESS_ITERS) + 255) / 256 * 256;
    VO_CUDA_CHECK(cudaMalloc(&ctx->d_unit_ess, (size_t)n_units * bytes));
    ctx->unit_ess_bytes = bytes; ctx->unit_ess_units = n_units;
    return VO_OK;
}

EssArgs vo_unit_ess_args(const vo_ctx* ctx, int u0, int n, int n_max, const int* count)
{
    EssArgs a;
    memset(&a, 0, sizeof(a));
    const size_t uo = (size_t)u0 * ctx->cap, cs = (size_t)ctx->units * ctx->cap;
    vo_ess_bind(a, (uint8_t*)ctx->d_unit_ess + (size_t)u0 * ctx->unit_ess_bytes, ctx->cap, VO_ESS_ITERS);
    a.n_max = n_max;
    a.n = count;
    a.cal = ctx->d_cal + u0;
    a.pts0 = ctx->d_valid4 + uo; a.pts1 = ctx->d_valid4 + 2 * cs + uo;
    a.n_prob = n;
    a.scratch_stride = a.result_stride = ctx->unit_ess_bytes; a.pts_stride = ctx->cap; a.n_stride = 1; a.cal_stride = 1;
    return a;
}

int vo_copy_unit_ess(vo_ctx* ctx, EssResult* dst, int u0, int n, cudaStream_t st)
{
    const EssArgs e = vo_unit_ess_args(ctx, u0, n, ctx->cap, nullptr);
    VO_CUDA_CHECK(cudaMemcpy2DAsync(dst, sizeof(EssResult), e.result, e.result_stride, sizeof(EssResult), n, cudaMemcpyDeviceToHost, st));
    return VO_OK;
}

vo_mono_result vo_mono_from_ess(const EssResult& e)
{
    vo_mono_result m;
    memset(&m, 0, sizeof(m));
    m.status = e.status == ESS_OK ? VO_OK : VO_E_TOO_FEW_POINTS;
    m.n_inliers = e.n_inliers; m.ransac_iters = e.iters; m.n_good = e.n_good;
    for (int k = 0; k < 9; k++) m.R[k] = e.R[k];
    for (int k = 0; k < 3; k++) m.t[k] = e.t[k];
    return m;
}

// entries [1 + u0, 1 + u0 + n) of a per-unit table (host copy `host`, device table `dev`)
template <typename T>
static int write_table(vo_ctx* ctx, std::vector<T>& host, T* dev, int u0, int n, const T* e)
{
    const size_t e0 = (size_t)(1 + u0);
    if (memcmp(host.data() + e0, e, n * sizeof(T)) == 0) return VO_OK;
    memcpy(host.data() + e0, e, n * sizeof(T));
    for (auto& p : ctx->pending)
        if (p.active) VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, p.done, 0));
    VO_CUDA_CHECK(cudaMemcpyAsync(dev + e0, host.data() + e0, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return VO_OK;
}

int vo_write_calib(vo_ctx* ctx, int u0, int n, const CamCalib* c) { return write_table(ctx, ctx->cal, ctx->d_cal_tab, u0, n, c); }

int vo_write_params(vo_ctx* ctx, int u0, int n, const UnitParams* e) { return write_table(ctx, ctx->par, ctx->d_par_tab, u0, n, e); }

int vo_set_calibration(vo_ctx* ctx, int u0, int n, const float* P_l, const float* P_r, int n_mat)
{
    std::vector<CamCalib> c(n);
    for (int i = 0; i < n; i++) c[i] = vo_calib_from(P_l + 12 * (i % n_mat), P_r + 12 * (i % n_mat));
    return vo_write_calib(ctx, u0, n, c.data());
}

void vo_free_state(vo_ctx* ctx)
{
    vo_drop_graphs(ctx);
    for (void* p : ctx->allocs) cudaFree(p);
    ctx->allocs.clear();
    if (ctx->d_seq_state) cudaFree(ctx->d_seq_state);
    ctx->d_seq_state = nullptr; ctx->seq_n_cap = 0;
    ctx->d_feat_pts = nullptr; ctx->d_feat_ages = nullptr; ctx->d_feat_cnt = ctx->d_bucket = ctx->d_seq_err = ctx->d_seq_live = nullptr;
    ctx->d_out = nullptr; ctx->out_stride = 0; ctx->out_per = 0;
    ctx->d_cal_tab = ctx->d_cal = nullptr;
    ctx->d_par_tab = ctx->d_par = nullptr;
    ctx->d_geo = nullptr;
    ctx->w = ctx->h = ctx->units = 0;
}

template <typename T>
static cudaError_t dalloc(vo_ctx* ctx, T** p, size_t count)
{
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, count * sizeof(T) + 256);
    if (e == cudaSuccess) { ctx->allocs.push_back(q); *p = (T*)q; }
    return e;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int encode_maps(vo_ctx* ctx)
{
    // resolved through the runtime so that the .so does not link libcuda (it must load on CPU-only hosts)
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    VO_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) {
        vo_set_error(ctx, "cuTensorMapEncodeTiled not available from the driver");
        return VO_E_CUDA;
    }
    PFN_encodeTiled enc = (PFN_encodeTiled)fn;
    const int n_img = ctx->units * 4;
    for (int l = 0; l < ctx->pg.nlevels; l++) {
        const LevelGeom& g = ctx->pg.lv[l];
        {
            cuuint64_t dims[3] = {(cuuint64_t)g.pitch, (cuuint64_t)g.hp, (cuuint64_t)n_img};
            cuuint64_t strides[2] = {(cuuint64_t)g.pitch, (cuuint64_t)g.plane};
            cuuint32_t box_i[3] = {48, 22, 1}, box_j[3] = {48, 32, 1};
            cuuint32_t estr[3] = {1, 1, 1};
            CUresult r = enc(&ctx->maps.img_i[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, g.img, dims, strides, box_i, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                             CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r == CUDA_SUCCESS)
                r = enc(&ctx->maps.img_j[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, g.img, dims, strides, box_j, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { vo_set_error(ctx, "cuTensorMapEncodeTiled(u8 level %d) failed: %d", l, (int)r); return VO_E_CUDA; }
        }
        {
            cuuint64_t dims[3] = {(cuuint64_t)g.pitch, (cuuint64_t)g.hp, (cuuint64_t)n_img};
            cuuint64_t strides[2] = {(cuuint64_t)g.pitch * 4, (cuuint64_t)g.plane * 4};
            cuuint32_t box[3] = {28, 22, 1};
            cuuint32_t estr[3] = {1, 1, 1};
            CUresult r = enc(&ctx->maps.der[l], CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, g.der, dims, strides, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                             CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { vo_set_error(ctx, "cuTensorMapEncodeTiled(deriv level %d) failed: %d", l, (int)r); return VO_E_CUDA; }
        }
    }
    return VO_OK;
}

int vo_ensure_state(vo_ctx* ctx, int w, int h, int units, int levels)
{
    if (w <= 0 || h <= 0 || units <= 0) { vo_set_error(ctx, "bad geometry %dx%d units=%d", w, h, units); return VO_E_INVALID; }
    const int depth = vo_pyr_depth(w, h, ctx->p.lk_max_level, ctx->p.lk_win);
    if (levels <= 0 || levels > depth) levels = depth;
    if (ctx->w == w && ctx->h == h && ctx->units >= units && ctx->pg.nlevels == levels) return VO_OK;
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    { int drc = vo_drain_pending(ctx); if (drc) return drc; }
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    vo_free_state(ctx);
    const int n_img = units * 4;
    const int cap = ctx->cap;
    // pyramid geometry: OpenCV stops adding levels once a level is not larger than the window
    PyrGeom& pg = ctx->pg;
    memset(&pg, 0, sizeof(pg));
    int cw = w, ch = h;
    for (int l = 0; l < levels; l++) {
        if (l > 0) { cw = (cw + 1) / 2; ch = (ch + 1) / 2; }
        LevelGeom& g = pg.lv[l];
        g.w = cw; g.h = ch;
        g.pitch = ((cw + 2 * VO_PAD) + 63) / 64 * 64;
        g.hp = ch + 2 * VO_PAD;
        g.plane = (size_t)g.pitch * g.hp;
        VO_CUDA_CHECK(dalloc(ctx, &g.img, g.plane * n_img));
        VO_CUDA_CHECK(dalloc(ctx, &g.der, g.plane * n_img));
        VO_CUDA_CHECK(cudaMemsetAsync(g.img, 0, g.plane * n_img, ctx->stream));
        VO_CUDA_CHECK(cudaMemsetAsync(g.der, 0, g.plane * n_img * sizeof(uint32_t), ctx->stream));
        pg.nlevels = l + 1;
    }
    pg.n_img = n_img;
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_raw, (size_t)n_img * w * h));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_raw_tab, (size_t)n_img));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_ingest_tab, (size_t)n_img));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_ingest_map, (size_t)n_img));
    {
        std::vector<const uint8_t*> tab(n_img);
        for (int i = 0; i < n_img; i++) tab[i] = ctx->d_raw + (size_t)i * w * h;
        VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_raw_tab, tab.data(), n_img * sizeof(uint8_t*), cudaMemcpyHostToDevice, ctx->stream));
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    }
    const size_t uc = (size_t)units * cap;
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_pts_in, uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_npts, (size_t)units));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_pts_out, 4 * uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_status, 4 * uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_err, 4 * uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_lk_progress, uc));
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_lk_progress, 0, uc * sizeof(int), ctx->stream));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_ages_in, uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_ages_out, uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_kept5, 5 * uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_idx3, uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_n3, (size_t)units));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_valid4, 4 * uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_idx5, uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_n5, (size_t)units));
    // FAST: room for every corner the frame can hold.  Corners lie in the (w-6) x (h-6) interior; under strict 3x3
    // non-max suppression two survivors are never 8-neighbours, so each 2x2 block holds at most one.
    {
        const long iw = w > 6 ? w - 6 : 0, ih = h > 6 ? h - 6 : 0;
        const long bound = ctx->p.fast_nonmax ? ((iw + 1) / 2) * ((ih + 1) / 2) : iw * ih;
        if (bound > (1L << 30)) { vo_set_error(ctx, "%dx%d: too many possible FAST corners", w, h); return VO_E_CAPACITY; }
        ctx->corner_cap = bound > 0 ? (int)bound : 1;
    }
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_score, (size_t)units * w * h));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_rowbuf, (size_t)units * h * w));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_rowcount, (size_t)units * h));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_rowoff, (size_t)units * h));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_ndet, (size_t)units));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_corners, (size_t)units * ctx->corner_cap));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_resp, (size_t)units * ctx->corner_cap));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_want, (size_t)units));
    // triangulation + PnP
    const size_t its = (size_t)vo_pnp_iterations(ctx);
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_X, uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_tprev, (size_t)units * 3));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_pnp_state, (size_t)units));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_subsets, (size_t)units * its * 5));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_models, (size_t)units * its * 12));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_counts, (size_t)units * its));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_inliers, uc));
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_results, (size_t)units));
    // calibration table: the entries set so far carry over (a unit keeps its camera until it is set again)
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_cal_tab, 1 + (size_t)units));
    ctx->d_cal = ctx->d_cal_tab + 1;
    ctx->cal.resize(1 + (size_t)units, CamCalib{});
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_cal_tab, ctx->cal.data(), (1 + (size_t)units) * sizeof(CamCalib), cudaMemcpyHostToDevice, ctx->stream));
    // parameter table: likewise; new entries (and entry 0, always) hold the context's vo_params
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_par_tab, 1 + (size_t)units));
    ctx->d_par = ctx->d_par_tab + 1;
    ctx->par.resize(1 + (size_t)units, vo_unit_params(ctx->p));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_par_tab, ctx->par.data(), (1 + (size_t)units) * sizeof(UnitParams), cudaMemcpyHostToDevice, ctx->stream));
    // sequence mode state: sized per sequence at vo_seq_begin / vo_mseq_begin (seq_api.cu)
    ctx->feat_cap = ctx->corner_cap + cap;
    ctx->seq_active = false;
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_results, 0, (size_t)units * sizeof(vo_unit_result_dev), ctx->stream));
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_tprev, 0, (size_t)units * 3 * sizeof(double), ctx->stream));
    ctx->w = w; ctx->h = h; ctx->units = units;
    // geometry table: every plane w x h until a run of several sizes writes its planes' entries
    VO_CUDA_CHECK(dalloc(ctx, &ctx->d_geo, (size_t)n_img));
    ctx->geo.assign((size_t)n_img, vo_plane_geom(ctx, w, h));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_geo, ctx->geo.data(), (size_t)n_img * sizeof(PlaneGeom), cudaMemcpyHostToDevice, ctx->stream));
    int rc = encode_maps(ctx);
    if (rc != VO_OK) { vo_free_state(ctx); return rc; }
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}

PlaneGeom vo_plane_geom(const vo_ctx* ctx, int w, int h)
{
    PlaneGeom g;
    memset(&g, 0, sizeof(g));
    for (int l = 0; l < ctx->pg.nlevels; l++) {
        g.w[l] = w; g.h[l] = h;
        w = (w + 1) / 2; h = (h + 1) / 2;
    }
    g.pitch = g.w[0];
    return g;
}

int vo_write_geo(vo_ctx* ctx, int p0, int n, const PlaneGeom* g, cudaStream_t st)
{
    if (memcmp(ctx->geo.data() + p0, g, n * sizeof(PlaneGeom)) == 0) return VO_OK;
    memcpy(ctx->geo.data() + p0, g, n * sizeof(PlaneGeom));
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_geo + p0, ctx->geo.data() + p0, n * sizeof(PlaneGeom), cudaMemcpyHostToDevice,
                                  st ? st : ctx->stream));
    return VO_OK;
}

// ---------------------------------------------------------------------------------------------
// pyramids (u8 + Scharr derivative, all levels) of the raw planes [plane0, plane0 + nplanes)
int vo_run_pyramid(vo_ctx* ctx, int plane0, int nplanes, cudaStream_t s, bool sized)
{
    PyrGeom pg = ctx->pg;
    pg.n_img = nplanes;
    for (int l = 0; l < pg.nlevels; l++) {
        pg.lv[l].img += (size_t)plane0 * pg.lv[l].plane;
        pg.lv[l].der += (size_t)plane0 * pg.lv[l].plane;
    }
    ctx->launches += vo_launch_pyramid(pg, ctx->d_raw_tab + plane0, ctx->w, sized ? ctx->d_geo + plane0 : nullptr, s);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

int vo_run_lk(vo_ctx* ctx, const View& v, int ncalls, const int* img_prev, const int* img_next, bool want_err, const UnitParams* par)
{
    int rc = vo_run_pyramid(ctx, v.u0 * v.imgs, v.n * v.imgs, v.s);
    if (rc) return rc;
    return vo_run_lk_ring(ctx, v, ncalls, img_prev, img_next, want_err, par);
}

// the ring kernel alone (pyramids of every plane it touches must be up to date)
int vo_run_lk_ring(vo_ctx* ctx, const View& v, int ncalls, const int* img_prev, const int* img_next, bool want_err,
                   const UnitParams* par)
{
    const size_t uo = (size_t)v.u0 * ctx->cap;
    const PyrGeom& pg = ctx->pg;

    LkArgs a;
    memset(&a, 0, sizeof(a));
    a.n_units = v.n;
    a.cap = ctx->cap;
    a.n_pts = ctx->d_npts + v.u0;
    a.imgs_per_unit = v.imgs;
    a.img_plane0 = v.plane0 >= 0 ? v.plane0 : v.u0 * v.imgs;
    a.ncalls = ncalls;
    for (int c = 0; c < ncalls; c++) { a.img_prev[c] = img_prev[c]; a.img_next[c] = img_next[c]; }
    a.nlevels = pg.nlevels;
    for (int l = 0; l < pg.nlevels; l++) { a.lw[l] = pg.lv[l].w; a.lh[l] = pg.lv[l].h; }
    a.geo = v.sized ? ctx->d_geo : nullptr;
    a.par = par + v.u0;
    a.pts_in = ctx->d_pts_in + uo;
    a.pts_out = ctx->d_pts_out + uo;
    a.status_out = ctx->d_status + uo;
    a.err_out = want_err ? ctx->d_err + uo : nullptr;
    a.call_stride = (size_t)ctx->units * ctx->cap;
    for (int l = 0; l < pg.nlevels; l++) {      // absolute plane bases (indexed with the absolute plane number)
        a.img_base[l] = ctx->pg.lv[l].img; a.der_base[l] = ctx->pg.lv[l].der;
        a.pitch[l] = pg.lv[l].pitch; a.plane[l] = pg.lv[l].plane;
    }

    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (ctx->lk_timing) {
        if (ctx->ev_used + 2 > ctx->ev_pool.size()) {
            cudaEvent_t a0, a1;
            VO_CUDA_CHECK(cudaEventCreate(&a0));
            VO_CUDA_CHECK(cudaEventCreate(&a1));
            ctx->ev_pool.push_back(a0); ctx->ev_pool.push_back(a1);
        }
        e0 = ctx->ev_pool[ctx->ev_used]; e1 = ctx->ev_pool[ctx->ev_used + 1];
        ctx->ev_used += 2;
        VO_CUDA_CHECK(cudaEventRecord(e0, v.s));
    }
    {
        // the queue pair of the launching stream
        size_t qi = 0;
        while (qi < ctx->lk_queue_streams.size() && ctx->lk_queue_streams[qi] != v.s) qi++;
        if (qi == ctx->lk_queue_streams.size()) {
            if (qi >= LK_QUEUES) { vo_set_error(ctx, "more than %d streams launch the LK kernel", LK_QUEUES); return VO_E_CAPACITY; }
            ctx->lk_queue_streams.push_back(v.s);
        }
        a.queue = ctx->d_lk_queue + 2 * qi;
        a.per_unit = v.max_pts > 0 && v.max_pts < ctx->cap ? v.max_pts : ctx->cap;
        a.progress = ctx->d_lk_progress + uo;
        int lk_sms = ctx->sm_count;
        for (const auto& L : ctx->lane) if (ctx->part_on && v.s == L.lk) lk_sms = ctx->part_lk_sms;
        if (ctx->p.lk_win != VO_WIN) {          // every other window: k_lk_win, one work item per feature-ring
            VO_CUDA_CHECK(vo_launch_lk_win(a, ctx->p.lk_win, lk_sms, v.s));
        } else {
            // a launch with fewer features than resident warps gains nothing from splitting its rings
            const bool big = (long)a.n_units * a.per_unit > (long)lk_sms * LK_CTAS_PER_SM * LK_WARPS_PER_CTA;
            a.span = ctx->lk_span > 0 ? ctx->lk_span : (big ? 2 : 0);
            VO_CUDA_CHECK(vo_launch_lk_ring(ctx->maps, a, lk_sms, v.s));
        }
    }
    ctx->launches += 1;
    if (e1) VO_CUDA_CHECK(cudaEventRecord(e1, v.s));
    return VO_OK;
}

int vo_run_filter(vo_ctx* ctx, const View& v, bool with_ages, const UnitParams* par)
{
    const size_t uo = (size_t)v.u0 * ctx->cap;
    FilterArgs f;
    memset(&f, 0, sizeof(f));
    f.cap = ctx->cap;
    f.call_stride = (size_t)ctx->units * ctx->cap;
    f.par = par + v.u0;
    f.n_pts = ctx->d_npts + v.u0;
    f.pts_in = ctx->d_pts_in + uo;
    f.pts_out = ctx->d_pts_out + uo;
    f.status = ctx->d_status + uo;
    f.ages_in = with_ages ? ctx->d_ages_in + uo : nullptr;
    f.ages_out = ctx->d_ages_out + uo;
    f.kept5 = ctx->d_kept5 + uo;
    f.idx3 = ctx->d_idx3 + uo;
    f.n3 = ctx->d_n3 + v.u0;
    f.valid4 = ctx->d_valid4 + uo;
    f.idx5 = ctx->d_idx5 + uo;
    f.n5 = ctx->d_n5 + v.u0;
    VO_CUDA_CHECK(vo_launch_ring_filter(f, v.n, v.s));
    ctx->launches += 1;
    return VO_OK;
}

int vo_run_fast(vo_ctx* ctx, const View& v, int plane_in_unit, bool want_resp, const UnitParams* par)
{
    FastArgs a;
    memset(&a, 0, sizeof(a));
    const size_t plane = (size_t)ctx->w * ctx->h;
    a.n_units = v.n;
    a.img_tab = ctx->d_raw_tab + (size_t)(v.plane0 >= 0 ? v.plane0 : v.u0 * v.imgs) + plane_in_unit;
    a.img_stride_idx = v.imgs;
    a.w = ctx->w; a.h = ctx->h; a.pitch = ctx->w;
    a.par = par + v.u0; a.nonmax = ctx->p.fast_nonmax;
    a.score = ctx->d_score + v.u0 * plane; a.score_plane = plane;
    a.rowbuf = ctx->d_rowbuf + v.u0 * plane; a.rowcap = ctx->w;
    a.rowcount = ctx->d_rowcount + (size_t)v.u0 * ctx->h; a.rowoff = ctx->d_rowoff + (size_t)v.u0 * ctx->h;
    a.n_det = ctx->d_ndet + v.u0;
    a.corners = ctx->d_corners + (size_t)v.u0 * ctx->corner_cap;
    a.resp = want_resp ? ctx->d_resp + (size_t)v.u0 * ctx->corner_cap : nullptr;
    a.corner_cap = ctx->corner_cap;
    a.geo = v.sized ? ctx->d_geo + (a.img_tab - ctx->d_raw_tab) : nullptr;
    ctx->launches += vo_launch_fast(a, v.s);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

int vo_run_select(vo_ctx* ctx, const View& v)
{
    ctx->launches += vo_launch_select(ctx->d_corners + (size_t)v.u0 * ctx->corner_cap, ctx->corner_cap, ctx->d_ndet + v.u0,
                                      ctx->d_want + v.u0, ctx->d_pts_in + (size_t)v.u0 * ctx->cap, ctx->cap, ctx->d_npts + v.u0,
                                      v.n, v.s);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

int vo_run_triangulate(vo_ctx* ctx, const View& v, const float2* pts_l, const float2* pts_r, const int* n, const CamCalib* cal,
                       float4* X4)
{
    const size_t uo = (size_t)v.u0 * ctx->cap;
    TriArgs t;
    memset(&t, 0, sizeof(t));
    t.cap = ctx->cap; t.n_pts = n + v.u0; t.pts_l = pts_l + uo; t.pts_r = pts_r + uo; t.X = ctx->d_X + uo; t.X4 = X4;
    t.cal = cal + v.u0;
    ctx->launches += vo_launch_triangulate(t, v.n, v.s);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

int vo_run_pnp(vo_ctx* ctx, const View& v, const float2* pts2d, const int* n, const CamCalib* cal, const UnitParams* par)
{
    const int iterations = vo_pnp_iterations(ctx);      // the stride of the RANSAC scratch; each unit runs its own count
    const size_t uo = (size_t)v.u0 * ctx->cap, its = (size_t)iterations;
    PnpArgs a;
    memset(&a, 0, sizeof(a));
    a.n_units = v.n; a.cap = ctx->cap; a.iterations = iterations;
    a.n_pts = n + v.u0; a.X = ctx->d_X + uo; a.x = pts2d + uo;
    a.cal = cal + v.u0;
    a.par = par + v.u0;
    a.t_prev = ctx->d_tprev + (size_t)v.u0 * 3;
    a.state = ctx->d_pnp_state + v.u0; a.subsets = ctx->d_subsets + v.u0 * its * 5; a.models = ctx->d_models + v.u0 * its * 12;
    a.counts = ctx->d_counts + v.u0 * its;
    a.inliers = ctx->d_inliers + uo; a.results = ctx->d_results + v.u0;
    ctx->launches += vo_launch_pnp(a, v.s);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}
