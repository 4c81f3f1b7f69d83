// seq_api.cu -- C-ABI of the streaming sequence mode (include/vo_b200.h, vo_seq_*).
//
// A pushed frame k is two stages on two streams:
//   front (the caller's stream):  upload of the new pair [-> BGR->gray] -> its two pyramids -> FAST refill on the previous
//        left image -> append + bucketing -> LK ring -> filters -> feature carry (currentVOFeatures = pointsLeft_t1)
//        -> triangulation
//   back  (a side stream):        PnP/RANSAC + LM from the carried translation -> translation carry -> result record to
//        pinned memory
// Only the back stage of frame k+1 needs the back stage of frame k (the extrinsic guess), so vo_seq_submit may be called
// for frame k+1 before vo_seq_wait returned frame k: its front stage then runs under the latency-bound pose solve of
// frame k.  Per-frame device buffers are the batch state's unit slots k & 1 (two frames in flight at most); the
// sequence state proper (FeatureSet, the image planes + pyramids, translation) is shared.  The stereo pairs live in a
// ring of THREE image slots (6 planes): gray uploads go through a copy stream into the slot that neither the running
// nor the previous frame reads, so the H2D of frame k+1 also runs under the kernels of frame k (double-buffered
// upload).  Each stage is one CUDA graph (per image-slot pair / buffer unit / input format).
//
// With the option "mono_rotation" (trackingFrame2Frame's header default, reference src/visualOdometry.cpp:146-157) the
// front stage also forks the essential-matrix RANSAC + recoverPose (ess.cu) onto seq_mono_stream as soon as the filters
// have compacted L0 / L1, so it runs beside the feature carry and the triangulation and is joined before the front stage
// ends; it reads no carried translation, so it stays off the back stage, whose PnP chain serialises consecutive frames.
// The back stage then writes recoverPose's rotation into the record (k_seq_mono); rvec / tvec / inliers stay the PnP's.
#include "ctx.h"
#include <string.h>

static int upload_pair(vo_ctx* ctx, int slot, const uint8_t* left, const uint8_t* right, size_t pitch, int channels, cudaStream_t st)
{
    const int w = ctx->w, h = ctx->h;
    const uint8_t* imgs[2] = {left, right};
    if (channels == 3) {                 // colour input: BGR bytes to the staging area, converted inside the frame's graph
        const size_t img = (size_t)3 * w * h;
        int rc = vo_ensure_bgr(ctx, 2 * img);
        if (rc) return rc;
        for (int k = 0; k < 2; k++)
            VO_CUDA_CHECK(cudaMemcpy2DAsync(ctx->d_bgr + k * img, (size_t)3 * w, imgs[k], pitch, (size_t)3 * w, h, cudaMemcpyHostToDevice, st));
        return VO_OK;
    }
    for (int k = 0; k < 2; k++) {
        uint8_t* dst = ctx->d_raw + (size_t)(2 * slot + k) * w * h;
        if (pitch == (size_t)w) VO_CUDA_CHECK(cudaMemcpyAsync(dst, imgs[k], (size_t)w * h, cudaMemcpyHostToDevice, st));
        else VO_CUDA_CHECK(cudaMemcpy2DAsync(dst, w, imgs[k], pitch, w, h, cudaMemcpyHostToDevice, st));
    }
    return VO_OK;
}

// BGR staging -> the two raw gray planes of `slot` (cv::cvtColor(BGR2GRAY) of utils.cpp:179,189)
static int convert_pair(vo_ctx* ctx, int slot)
{
    const int w = ctx->w, h = ctx->h;
    ctx->launches += vo_launch_bgr_to_gray(nullptr, vo_packed_bgr(ctx->d_bgr, w), (size_t)3 * w * h, ctx->d_raw + (size_t)(2 * slot) * w * h,
                                           (size_t)w * h, w, h, 2, ctx->stream);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

static void seq_args(vo_ctx* ctx, int unit, SeqArgs& a)
{
    memset(&a, 0, sizeof(a));
    const size_t uo = (size_t)unit * ctx->cap, cs = (size_t)ctx->units * ctx->cap;
    a.corners = ctx->d_corners + (size_t)unit * ctx->corner_cap; a.n_det = ctx->d_ndet + unit; a.corner_cap = ctx->corner_cap;
    a.feat_pts = ctx->d_feat_pts; a.feat_ages = ctx->d_feat_ages; a.cnt = ctx->d_feat_cnt; a.feat_cap = ctx->feat_cap;
    a.refill_below = 2000;                                   // visualOdometry.cpp:95
    a.rows = ctx->h; a.cols = ctx->w; a.bucket_size = ctx->h / 10;      // visualOdometry.cpp:106 (features_per_bucket = 1)
    a.bucket = ctx->d_bucket; a.bucket_cap = ctx->bucket_cap;
    a.out_pts = ctx->d_pts_in + uo; a.out_ages = ctx->d_ages_in + uo; a.out_n = ctx->d_npts + unit; a.out_cap = ctx->cap;
    a.valid_l1 = ctx->d_valid4 + 2 * cs + uo; a.n5 = ctx->d_n5 + unit; a.ages_out = ctx->d_ages_out + uo; a.n3 = ctx->d_n3 + unit;
    a.res = ctx->d_results + unit;
    a.tprev = ctx->d_tprev + 3 * (size_t)(1 - unit);          // the next frame solves from this frame's translation
    a.err = ctx->d_seq_err + 1 + unit; a.err_out = ctx->d_seq_err + 1 + unit;      // one word per buffer unit = per frame in flight
}

// bucketingFeatures() reads back (rows/bs + 1) x (cols/bs + 1) slots at most (feature.cpp:242-249): the bound of every
// per-frame point count
static int seq_grid(const vo_ctx* ctx)
{
    const int bs = ctx->h / 10 > 0 ? ctx->h / 10 : 1;
    return (ctx->h / bs + 1) * (ctx->w / bs + 1);
}

// the mono branch of buffer unit `unit`: pointsLeft_t0 / pointsLeft_t1 = the filtered L0 / L1 lists (d_valid4 planes 0, 2)
static void seq_ess_args(vo_ctx* ctx, int unit, EssArgs& a)
{
    memset(&a, 0, sizeof(a));
    const size_t uo = (size_t)unit * ctx->cap, cs = (size_t)ctx->units * ctx->cap;
    // `double focal = projMatrl.at<float>(0, 0)`, principle_point(projMatrl.at<float>(0, 2), projMatrl.at<float>(1, 2))
    vo_ess_set_camera(a, (double)ctx->P_l[0], (double)ctx->P_l[2], (double)ctx->P_l[6]);
    vo_ess_bind(a, (uint8_t*)ctx->d_seq_ess + (size_t)unit * ctx->seq_ess_bytes, ctx->seq_ess_cap, VO_ESS_ITERS);
    a.n = ctx->d_n5 + unit;
    a.pts0 = ctx->d_valid4 + uo; a.pts1 = ctx->d_valid4 + 2 * cs + uo;
}

// per-unit scratch of the mono branch, sized for the bucket grid (outside any capture: vo_seq_begin)
static int seq_mono_scratch(vo_ctx* ctx)
{
    const int grid = seq_grid(ctx);
    const int n_max = grid < ctx->cap ? grid : ctx->cap;
    if (!ctx->seq_mono_stream) {
        VO_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->seq_mono_stream, cudaStreamNonBlocking));
        for (int k = 0; k < 2; k++) VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->seq_mono_ev[k], cudaEventDisableTiming));
    }
    if (ctx->d_seq_ess && ctx->seq_ess_cap >= n_max) return VO_OK;
    vo_drop_graphs(ctx);                                      // captured graphs hold the old blocks
    if (ctx->d_seq_ess) { VO_CUDA_CHECK(cudaDeviceSynchronize()); cudaFree(ctx->d_seq_ess); ctx->d_seq_ess = nullptr; }
    const size_t bytes = (vo_ess_scratch_bytes(n_max, VO_ESS_ITERS) + 255) / 256 * 256;
    VO_CUDA_CHECK(cudaMalloc(&ctx->d_seq_ess, 2 * bytes));
    ctx->seq_ess_bytes = bytes; ctx->seq_ess_cap = n_max;
    return VO_OK;
}

static const EssResult* seq_ess_result(vo_ctx* ctx, int unit)
{
    EssArgs a;
    seq_ess_args(ctx, unit, a);
    return a.result;
}

// front stage of one frame on the caller's stream; s0 / s1 = image slots of the previous / new pair, unit = per-frame buffers
static int seq_front(vo_ctx* ctx, int s0, int s1, int unit, bool bgr)
{
    ctx->imgs_per_unit = 4;
    const int L0 = 2 * s0, R0 = 2 * s0 + 1, L1 = 2 * s1, R1 = 2 * s1 + 1;
    const View v{unit, 1, ctx->stream, 0};                    // image planes are 0..5 whatever the buffer unit
    int rc;
    if (bgr && (rc = convert_pair(ctx, s1))) return rc;
    // the new pair's two pyramids (the previous pair's are already resident)
    if ((rc = vo_run_pyramid(ctx, 2 * s1, 2, ctx->stream))) return rc;
    // matchingFeatures(): FAST refill on the t0 left image -> bucketing -> circular matching -> filters
    if ((rc = vo_run_fast(ctx, v, L0, false))) return rc;
    SeqArgs a;
    seq_args(ctx, unit, a);
    ctx->launches += vo_launch_seq_append(a, ctx->stream);
    ctx->launches += vo_launch_seq_bucket(a, ctx->stream);
    const int ip[4] = {L0, R0, R1, L1}, in[4] = {R0, R1, L1, L0};
    ctx->lk_per_unit = seq_grid(ctx);
    rc = vo_run_lk_ring(ctx, v, 4, ip, in, false);
    ctx->lk_per_unit = 0;
    if (rc) return rc;
    if ((rc = vo_run_filter(ctx, v, true))) return rc;
    if (ctx->seq_mono) {        // findEssentialMat + recoverPose on (L0, L1), beside the carry and the triangulation
        EssArgs e;
        seq_ess_args(ctx, unit, e);
        VO_CUDA_CHECK(cudaEventRecord(ctx->seq_mono_ev[0], ctx->stream));
        VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->seq_mono_stream, ctx->seq_mono_ev[0], 0));
        ctx->launches += vo_launch_essential(e, ctx->seq_mono_stream);
        VO_CUDA_CHECK(cudaGetLastError());
        VO_CUDA_CHECK(cudaEventRecord(ctx->seq_mono_ev[1], ctx->seq_mono_stream));
    }
    // state carry: features.points = pointsLeft_t1, ages keep their A3 length
    ctx->launches += vo_launch_seq_carry(a, ctx->stream);
    const size_t cs = (size_t)ctx->units * ctx->cap;
    if ((rc = vo_run_triangulate(ctx, v, ctx->d_valid4, ctx->d_valid4 + cs, ctx->d_n5))) return rc;
    if (ctx->seq_mono) VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->seq_mono_ev[1], 0));
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

// back stage on side stream 0: trackingFrame2Frame's PnP + translation carry (+ the mono rotation into the record)
static int seq_back(vo_ctx* ctx, int unit)
{
    cudaStream_t st = ctx->side_stream[0];
    const View v{unit, 1, st, 0};
    const size_t cs = (size_t)ctx->units * ctx->cap;
    float K9[9] = {ctx->P_l[0], ctx->P_l[1], ctx->P_l[2], ctx->P_l[4], ctx->P_l[5], ctx->P_l[6], ctx->P_l[8], ctx->P_l[9], ctx->P_l[10]};
    int rc;
    if ((rc = vo_run_pnp(ctx, v, ctx->d_valid4 + 2 * cs, ctx->d_n5, K9))) return rc;
    SeqArgs a;
    seq_args(ctx, unit, a);
    ctx->launches += vo_launch_seq_finish(a, st);
    if (ctx->seq_mono) ctx->launches += vo_launch_seq_mono(ctx->d_results + unit, seq_ess_result(ctx, unit), st);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

// replay (or first capture) one stage as a CUDA graph on stream `st`
template <typename F>
static int seq_graph(vo_ctx* ctx, int key, cudaStream_t st, F launch)
{
    if (!ctx->use_graphs) return launch();
    for (auto& g : ctx->graphs)
        if (g.u0 == key && g.tma == ctx->lk_use_tma && g.s == st) {
            VO_CUDA_CHECK(cudaGraphLaunch(g.exec, st));
            ctx->launches += g.launches;
            return VO_OK;
        }
    const bool timing = ctx->lk_timing;
    const long long before = ctx->launches;
    ctx->lk_timing = false;
    cudaGraph_t graph = nullptr;
    VO_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    int rc = launch();
    cudaError_t e = cudaStreamEndCapture(st, &graph);
    ctx->lk_timing = timing;
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    VO_CUDA_CHECK(e);
    vo_ctx::RangeGraph g;
    g.u0 = key; g.n = 1; g.detect = true; g.tma = ctx->lk_use_tma; g.s = st; g.max_pts = 0;
    g.launches = ctx->launches - before;
    VO_CUDA_CHECK(cudaGraphInstantiate(&g.exec, graph, 0));
    cudaGraphDestroy(graph);
    ctx->graphs.push_back(g);
    VO_CUDA_CHECK(cudaGraphLaunch(g.exec, st));
    return VO_OK;
}

struct SeqRecord { vo_unit_result_dev r; int err; int pad_[3]; EssResult ess; /* mono sequences only */ };
// pinned staging of the sequence mode: SeqRecord[2] (one per buffer unit) | vo_dimage[6] (device-image descriptors, one per
// raw plane of the three-slot ring; plane 2s + k is restaged only after the frame that last used it has been waited for)
static const size_t SEQ_PINNED_BYTES = 2 * sizeof(SeqRecord) + 6 * sizeof(vo_dimage) + 256;
static vo_dimage* seq_pinned_tab(vo_ctx* ctx) { return (vo_dimage*)((SeqRecord*)ctx->h_pinned + 2); }

static int seq_events(vo_ctx* ctx)
{
    if (ctx->seq_front_ev[0]) return VO_OK;
    for (int k = 0; k < 2; k++) {
        VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->seq_front_ev[k], cudaEventDisableTiming));
        VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->seq_back_ev[k], cudaEventDisableTiming));
    }
    if (!ctx->side_stream[0]) {
        VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->fork_ev, cudaEventDisableTiming));
        for (int c = 0; c < VO_LANES; c++) {
            VO_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->side_stream[c], cudaStreamNonBlocking));
            VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->join_ev[c], cudaEventDisableTiming));
        }
    }
    return VO_OK;
}

// retire every frame in flight without reporting it (state queries / re-begin / destroy)
static int seq_drain(vo_ctx* ctx)
{
    if (ctx->seq_inflight > 0) {
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->side_stream[0]));
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    }
    return VO_OK;
}

extern "C" int vo_seq_begin(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const uint8_t* left0,
                            const uint8_t* right0, size_t pitch)
{
    return vo_seq_begin_ex(ctx, w, h, P_l, P_r, left0, right0, pitch, 1);
}

// a new sequence whose first pair `fill_slot0` enqueues into image slot 0 on ctx->stream (arguments already checked)
template <typename F>
static int seq_begin(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], F fill_slot0)
{
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    int rc;
    if (ctx->seq_active && (rc = seq_drain(ctx))) return rc;
    ctx->seq_inflight = 0;
    if ((rc = vo_ensure_state(ctx, w, h, 2, 4))) return rc;          // two per-frame buffer units (frames in flight)
    if ((rc = seq_events(ctx))) return rc;
    // the option holds for the whole sequence; the frame graphs are captured with or without the branch
    if (ctx->seq_mono != ctx->mono_opt) { vo_drop_graphs(ctx); ctx->seq_mono = ctx->mono_opt; }
    if (ctx->seq_mono && (rc = seq_mono_scratch(ctx))) return rc;
    if ((rc = vo_ensure_pinned(ctx, SEQ_PINNED_BYTES))) return rc;
    vo_set_calibration(ctx, P_l, P_r);
    ctx->imgs_per_unit = 4;
    ctx->seq_slot = 0;
    ctx->seq_frames = 0;
    ctx->seq_submitted = 0;
    for (int i = 0; i < 16; i++) ctx->seq_pose[i] = (i % 5 == 0) ? 1.0 : 0.0;
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_feat_cnt, 0, 2 * sizeof(int), ctx->stream));
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_seq_err, 0, 4 * sizeof(int), ctx->stream));
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_tprev, 0, 6 * sizeof(double), ctx->stream));      // translation = zeros (main.cpp:82)
    if ((rc = fill_slot0())) return rc;
    if ((rc = vo_run_pyramid(ctx, 0, 2, ctx->stream))) return rc;
    // both event pairs start out signalled, so the first two frames do not wait for a predecessor
    for (int k = 0; k < 2; k++) {
        VO_CUDA_CHECK(cudaEventRecord(ctx->seq_front_ev[k], ctx->stream));
        VO_CUDA_CHECK(cudaEventRecord(ctx->seq_back_ev[k], ctx->stream));
    }
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->seq_active = true;
    return VO_OK;
}

extern "C" int vo_seq_begin_ex(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const uint8_t* left0,
                               const uint8_t* right0, size_t pitch, int channels)
{
    if (!ctx) return VO_E_INVALID;
    if (channels != 1 && channels != 3) { vo_set_error(ctx, "vo_seq_begin: channels must be 1 (gray) or 3 (BGR)"); return VO_E_INVALID; }
    if (!P_l || !P_r || !left0 || !right0 || w <= 0 || h <= 0 || pitch < (size_t)w * channels) { vo_set_error(ctx, "vo_seq_begin: bad argument"); return VO_E_INVALID; }
    if (h / 10 <= 0) { vo_set_error(ctx, "vo_seq_begin: image too small for the rows/10 bucket size"); return VO_E_UNSUPPORTED; }
    return seq_begin(ctx, w, h, P_l, P_r, [&] {
        int rc = upload_pair(ctx, 0, left0, right0, pitch, channels, ctx->stream);
        return rc ? rc : channels == 3 ? convert_pair(ctx, 0) : VO_OK;
    });
}

extern "C" int vo_seq_begin_device(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const vo_dimage* left0,
                                   const vo_dimage* right0)
{
    if (!ctx) return VO_E_INVALID;
    if (!P_l || !P_r || w <= 0 || h <= 0) { vo_set_error(ctx, "vo_seq_begin_device: bad argument"); return VO_E_INVALID; }
    int rc;
    if ((rc = vo_check_dimage(ctx, "vo_seq_begin_device", "left0", left0, w)) || (rc = vo_check_dimage(ctx, "vo_seq_begin_device", "right0", right0, w))) return rc;
    if (h / 10 <= 0) { vo_set_error(ctx, "vo_seq_begin_device: image too small for the rows/10 bucket size"); return VO_E_UNSUPPORTED; }
    // on the caller's stream, after the work already enqueued there; vo_seq_begin ends with a synchronise (the release)
    return seq_begin(ctx, w, h, P_l, P_r, [&] {
        vo_dimage* tab = seq_pinned_tab(ctx);
        tab[0] = *left0; tab[1] = *right0;
        return vo_ingest_device(ctx, tab, 2, 0, ctx->stream);
    });
}

static int seq_enqueue(vo_ctx* ctx, int unit, int s0, int s1, bool bgr);

extern "C" int vo_seq_submit(vo_ctx* ctx, const uint8_t* left1, const uint8_t* right1, size_t pitch, int channels)
{
    if (!ctx) return VO_E_INVALID;
    if (channels != 1 && channels != 3) { vo_set_error(ctx, "vo_seq_submit: channels must be 1 (gray) or 3 (BGR)"); return VO_E_INVALID; }
    if (!ctx->seq_active) { vo_set_error(ctx, "vo_seq_submit: call vo_seq_begin first"); return VO_E_INVALID; }
    if (!left1 || !right1 || pitch < (size_t)ctx->w * channels) { vo_set_error(ctx, "vo_seq_submit: bad argument"); return VO_E_INVALID; }
    if (ctx->seq_inflight >= 2) { vo_set_error(ctx, "vo_seq_submit: two frames are in flight already; call vo_seq_wait"); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const int unit = (int)(ctx->seq_submitted & 1);
    const int s0 = ctx->seq_slot, s1 = (s0 + 1) % 3;
    const bool bgr = channels == 3;
    int rc;
    // the per-frame buffers of `unit` were last read by the back stage of frame k-2
    VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->seq_back_ev[unit], 0));
    if (bgr) {
        // colour frames share one staging buffer: upload + convert stay on the front stream
        if ((rc = upload_pair(ctx, s1, left1, right1, pitch, channels, ctx->stream))) return rc;
    } else {
        // image slot s1 (of three) was last read, as the previous pair, by the front stage of the frame before the one
        // now running: that frame has this frame's buffer parity, and its seq_front_ev[unit] record is still the
        // current one (it is re-recorded below).  So this copy runs under the front stage of the frame in flight.
        // (No ordering against the caller's stream is needed: vo_seq_begin synchronises, and every later access to
        // the image slots is made by this file and ordered through these events.)
        cudaStream_t sc = ctx->side_stream[1];
        VO_CUDA_CHECK(cudaStreamWaitEvent(sc, ctx->seq_front_ev[unit], 0));
        if ((rc = upload_pair(ctx, s1, left1, right1, pitch, channels, sc))) return rc;
        VO_CUDA_CHECK(cudaEventRecord(ctx->join_ev[1], sc));
        VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->join_ev[1], 0));
    }
    return seq_enqueue(ctx, unit, s0, s1, bgr);
}

// The rest of vo_seq_submit[_device] once the new pair is (being) written into image slot s1: the front stage (gray frames
// replay the gray graph whatever their source), the back stage, the record copies
static int seq_enqueue(vo_ctx* ctx, int unit, int s0, int s1, bool bgr)
{
    int rc;
    if ((rc = seq_graph(ctx, -1 - (s0 + 3 * unit + 6 * (bgr ? 1 : 0)), ctx->stream, [&] { return seq_front(ctx, s0, s1, unit, bgr); }))) return rc;
    VO_CUDA_CHECK(cudaEventRecord(ctx->seq_front_ev[unit], ctx->stream));
    // back stage: after this frame's front stage; after the previous frame's back stage by stream order
    cudaStream_t sb = ctx->side_stream[0];
    VO_CUDA_CHECK(cudaStreamWaitEvent(sb, ctx->seq_front_ev[unit], 0));
    if ((rc = seq_graph(ctx, -100 - unit, sb, [&] { return seq_back(ctx, unit); }))) return rc;
    SeqRecord* rec = (SeqRecord*)ctx->h_pinned + unit;
    VO_CUDA_CHECK(cudaMemcpyAsync(&rec->r, ctx->d_results + unit, sizeof(rec->r), cudaMemcpyDeviceToHost, sb));
    VO_CUDA_CHECK(cudaMemcpyAsync(&rec->err, ctx->d_seq_err + 1 + unit, sizeof(int), cudaMemcpyDeviceToHost, sb));
    if (ctx->seq_mono) VO_CUDA_CHECK(cudaMemcpyAsync(&rec->ess, seq_ess_result(ctx, unit), sizeof(rec->ess), cudaMemcpyDeviceToHost, sb));
    VO_CUDA_CHECK(cudaEventRecord(ctx->seq_back_ev[unit], sb));
    ctx->seq_slot = s1;                 // imageLeft_t0 = imageLeft_t1 (main.cpp:157-158)
    ctx->seq_channels[unit] = bgr ? 3 : 1;
    ctx->seq_submitted++;
    ctx->seq_inflight++;
    return VO_OK;
}

extern "C" int vo_seq_submit_device(vo_ctx* ctx, const vo_dimage* left1, const vo_dimage* right1)
{
    if (!ctx) return VO_E_INVALID;
    if (!ctx->seq_active) { vo_set_error(ctx, "vo_seq_submit_device: call vo_seq_begin first"); return VO_E_INVALID; }
    int rc;
    if ((rc = vo_check_dimage(ctx, "vo_seq_submit_device", "left1", left1, ctx->w)) ||
        (rc = vo_check_dimage(ctx, "vo_seq_submit_device", "right1", right1, ctx->w))) return rc;
    if (ctx->seq_inflight >= 2) { vo_set_error(ctx, "vo_seq_submit_device: two frames are in flight already; call vo_seq_wait"); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const int unit = (int)(ctx->seq_submitted & 1);
    const int s0 = ctx->seq_slot, s1 = (s0 + 1) % 3;
    // Producer ordering: the conversion reads the images after the caller's work enqueued so far.  The event is recorded
    // BEFORE the front stream waits for frame k-2's back stage below, so that the conversion does not queue behind that
    // pose solve.
    VO_CUDA_CHECK(cudaEventRecord(ctx->fork_ev, ctx->stream));
    VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->seq_back_ev[unit], 0));
    // As the host gray upload: on the copy stream, into slot s1 once the frame that last read it has finished its front
    // stage, so the conversion runs under the frame in flight; it is launched outside the frame graph (its source pointers
    // change every frame), and the frame replays the gray front graph.
    cudaStream_t sc = ctx->side_stream[1];
    VO_CUDA_CHECK(cudaStreamWaitEvent(sc, ctx->seq_front_ev[unit], 0));
    VO_CUDA_CHECK(cudaStreamWaitEvent(sc, ctx->fork_ev, 0));
    vo_dimage* tab = seq_pinned_tab(ctx) + 2 * s1;
    tab[0] = *left1; tab[1] = *right1;
    if ((rc = vo_ingest_device(ctx, tab, 2, 2 * s1, sc))) return rc;
    // The join is also the release: the caller's later work on ctx->stream is ordered after the conversion, the last read
    // of the images.
    VO_CUDA_CHECK(cudaEventRecord(ctx->join_ev[1], sc));
    VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->join_ev[1], 0));
    return seq_enqueue(ctx, unit, s0, s1, false);
}

static int seq_wait(vo_ctx* ctx, vo_unit_result* out, vo_mono_result* mono, uint8_t* ess_mask, int mask_cap, vo_point2f* pts4,
                    int pts_cap)
{
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const int unit = (int)((ctx->seq_submitted - ctx->seq_inflight) & 1);      // the oldest frame in flight
    VO_CUDA_CHECK(cudaEventSynchronize(ctx->seq_back_ev[unit]));
    const SeqRecord rec = *((const SeqRecord*)ctx->h_pinned + unit);
    memcpy(out, &rec.r, sizeof(rec.r));
    ctx->seq_inflight--;
    ctx->seq_frames++;
    // main.cpp:196-208.  The reference ignores solvePnPRansac's return value: when RANSAC finds no model, rvec stays 0
    // (R = I) and `translation` keeps the carried value, and the main loop still integrates that motion.  With
    // mono_rotation, where cv::findEssentialMat / cv::recoverPose would throw (n < 5, no E with more than 4 inliers,
    // n == 5 with other than one candidate) the frame is reported (R = I) and not integrated, like an n < 4 PnP frame.
    const bool mono_ok = !ctx->seq_mono || rec.ess.status == ESS_OK;
    if ((rec.r.pnp_status == VO_OK || rec.r.pnp_status == VO_PNP_NO_MODEL) && mono_ok) vo_pose_step(ctx->seq_pose, rec.r.R, rec.r.tvec);
    if (mono) {
        mono->status = mono_ok ? VO_OK : VO_E_TOO_FEW_POINTS;
        mono->n_inliers = rec.ess.n_inliers; mono->ransac_iters = rec.ess.iters; mono->n_good = rec.ess.n_good;
        for (int k = 0; k < 9; k++) mono->R[k] = rec.ess.R[k];
        for (int k = 0; k < 3; k++) mono->t[k] = rec.ess.t[k];
    }
    // the frame's point lists (and essential mask) stay in its buffer unit until the frame after next is submitted
    const bool want_pts = pts4 && pts_cap > 0 && rec.r.n_valid > 0, want_mask = ess_mask && mask_cap > 0 && rec.r.n_valid > 0;
    if (want_pts || want_mask) {
        const size_t cs = (size_t)ctx->units * ctx->cap, uo = (size_t)unit * ctx->cap;
        cudaStream_t sb = ctx->side_stream[0];
        if (want_pts) {
            const int n = rec.r.n_valid < pts_cap ? rec.r.n_valid : pts_cap;
            for (int k = 0; k < 4; k++)
                VO_CUDA_CHECK(cudaMemcpyAsync(pts4 + (size_t)k * pts_cap, ctx->d_valid4 + k * cs + uo, (size_t)n * sizeof(float2), cudaMemcpyDeviceToHost, sb));
        }
        if (want_mask) {
            EssArgs e;
            seq_ess_args(ctx, unit, e);
            const int n = rec.r.n_valid < mask_cap ? rec.r.n_valid : mask_cap;
            VO_CUDA_CHECK(cudaMemcpyAsync(ess_mask, e.mask, (size_t)n, cudaMemcpyDeviceToHost, sb));
        }
        VO_CUDA_CHECK(cudaStreamSynchronize(sb));
    }
    // bit 8 (a tracked point outside the bucket grid: undefined behaviour in the reference, dropped here) is not an error
    if (rec.err & ~8) { vo_set_error(ctx, "vo_seq: glue kernel error bits 0x%x of this frame (1/2: capacity, 4: bucket grid)", rec.err); return VO_E_CAPACITY; }
    return VO_OK;
}

extern "C" int vo_seq_wait(vo_ctx* ctx, vo_unit_result* out, vo_point2f* pts4, int pts_cap)
{
    if (!ctx) return VO_E_INVALID;
    if (!ctx->seq_active || ctx->seq_inflight <= 0) { vo_set_error(ctx, "vo_seq_wait: no frame in flight"); return VO_E_INVALID; }
    if (!out) { vo_set_error(ctx, "vo_seq_wait: null result"); return VO_E_INVALID; }
    return seq_wait(ctx, out, nullptr, nullptr, 0, pts4, pts_cap);
}

extern "C" int vo_seq_wait_mono(vo_ctx* ctx, vo_unit_result* out, vo_mono_result* mono, uint8_t* ess_mask, int mask_cap,
                                vo_point2f* pts4, int pts_cap)
{
    if (!ctx) return VO_E_INVALID;
    if (!ctx->seq_active || ctx->seq_inflight <= 0) { vo_set_error(ctx, "vo_seq_wait_mono: no frame in flight"); return VO_E_INVALID; }
    if (!out || !mono) { vo_set_error(ctx, "vo_seq_wait_mono: null result"); return VO_E_INVALID; }
    if (!ctx->seq_mono) { vo_set_error(ctx, "vo_seq_wait_mono: the sequence was begun without the option \"mono_rotation\""); return VO_E_INVALID; }
    return seq_wait(ctx, out, mono, ess_mask, mask_cap, pts4, pts_cap);
}

extern "C" int vo_seq_push(vo_ctx* ctx, const uint8_t* left1, const uint8_t* right1, size_t pitch, vo_unit_result* out,
                           vo_point2f* pts4, int pts_cap)
{
    return vo_seq_push_ex(ctx, left1, right1, pitch, 1, out, pts4, pts_cap);
}

// synchronous form: submit + wait (no other frame may be in flight)
extern "C" int vo_seq_push_ex(vo_ctx* ctx, const uint8_t* left1, const uint8_t* right1, size_t pitch, int channels,
                              vo_unit_result* out, vo_point2f* pts4, int pts_cap)
{
    if (!ctx) return VO_E_INVALID;
    if (!out) { vo_set_error(ctx, "vo_seq_push: null result"); return VO_E_INVALID; }
    if (ctx->seq_inflight != 0) { vo_set_error(ctx, "vo_seq_push: frames submitted with vo_seq_submit are still in flight"); return VO_E_INVALID; }
    int rc = vo_seq_submit(ctx, left1, right1, pitch, channels);
    if (rc) return rc;
    return vo_seq_wait(ctx, out, pts4, pts_cap);
}

extern "C" int vo_seq_state(vo_ctx* ctx, vo_point2f* points, int32_t* ages, int cap, int* n_points, int* n_ages, double t_out[3])
{
    if (!ctx || !ctx->seq_active) return VO_E_INVALID;
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    int rc = seq_drain(ctx);
    if (rc) return rc;
    int cnt[2] = {0, 0};
    VO_CUDA_CHECK(cudaMemcpyAsync(cnt, ctx->d_feat_cnt, 2 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    // the translation the NEXT frame will start from lives in the next frame's buffer unit
    if (t_out) VO_CUDA_CHECK(cudaMemcpyAsync(t_out, ctx->d_tprev + 3 * (size_t)(ctx->seq_submitted & 1), 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (n_points) *n_points = cnt[0];
    if (n_ages) *n_ages = cnt[1];
    if (points && cnt[0] > 0) VO_CUDA_CHECK(cudaMemcpyAsync(points, ctx->d_feat_pts, (size_t)(cnt[0] < cap ? cnt[0] : cap) * sizeof(float2), cudaMemcpyDeviceToHost, ctx->stream));
    if (ages && cnt[1] > 0) VO_CUDA_CHECK(cudaMemcpyAsync(ages, ctx->d_feat_ages, (size_t)(cnt[1] < cap ? cnt[1] : cap) * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}
