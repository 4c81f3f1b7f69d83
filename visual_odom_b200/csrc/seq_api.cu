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
// vo_mseq_* runs n_seq independent sequences (each with its own calibration: the kernels read unit u's camera from the
// calibration table, and sequence q's entries are those of units q and n_seq + q; and each with its own image size:
// vo_mseq_begin_sized) in lockstep through the same two stages:
// every stage kernel takes the n_seq units of a buffer parity (sequence q at parity p is unit p * n_seq + q) in ONE launch,
// and vo_seq_* is the same code with n_seq = 1.  The image ring is slot-major: slot s holds the pairs of all sequences,
// planes 2 * n_seq * s + 2q (left) and + 1 (right), so the new pairs of a frame are one contiguous run of planes (one
// pyramid launch, one BGR conversion) and FAST / the LK ring address sequence q's planes with an image stride of 2.
// Sequences of several image sizes share planes allocated at the envelope of the sizes (the largest width and height);
// each image's rows are packed from its plane's start, the geometry table (vo_ctx::d_geo) holds every plane's own size,
// and the pyramid, FAST, LK ring, BGR conversion and bucketing kernels read it (View::sized, SeqArgs::geo).  The table
// lives with the batch state, so the frame graphs carry no sizes; with one size the kernels take no table at all.
//
// With the option "mono_rotation" (vo_seq_*) or the flag VO_MSEQ_MONO_ROTATION (vo_mseq_begin_ex) -- trackingFrame2Frame's
// header default, reference src/visualOdometry.cpp:146-157 -- the front stage also forks the essential-matrix RANSAC +
// recoverPose (ess.cu) onto seq_mono_stream as soon as the filters have compacted L0 / L1: one launch sequence for the
// n_seq units of the parity (one problem per sequence), which runs beside the feature carry and the triangulation and is
// joined before the front stage ends; it reads no carried translation, so it stays off the back stage, whose PnP chain
// serialises consecutive frames.  The back stage then writes each sequence's recoverPose rotation into its record
// (k_seq_mono); rvec / tvec / inliers stay the PnP's.
#include "ctx.h"
#include <string.h>
#include <algorithm>

// the new host pairs of image slot `slot` (sequence q: lefts[q], rights[q]; a NULL pair is skipped): gray into the raw
// planes, colour (BGR) bytes into the staging area, converted inside the frame's graph
// planes (a staging image holds an envelope plane's pixels); every image goes with its own rows of its own width, pitch[q]
// bytes apart in host memory
static int upload_pairs(vo_ctx* ctx, int slot, const uint8_t* const* lefts, const uint8_t* const* rights, const size_t* pitch,
                        int channels, cudaStream_t st)
{
    const int n = ctx->seq_n;
    const size_t img = (size_t)channels * ctx->w * ctx->h;
    uint8_t* dst = ctx->d_raw + (size_t)(2 * n * slot) * ctx->w * ctx->h;
    int rc;
    if (channels == 3) {
        if ((rc = vo_ensure_bgr(ctx, 2 * (size_t)n * img))) return rc;
        dst = ctx->d_bgr;
    }
    for (int q = 0; q < n; q++) {
        if (!lefts[q]) continue;
        const uint8_t* imgs[2] = {lefts[q], rights[q]};
        for (int k = 0; k < 2; k++)
            if ((rc = vo_upload_plane(ctx, dst + (2 * q + k) * img, imgs[k], (size_t)channels * ctx->seq_w[q], ctx->seq_h[q], pitch[q], st)))
                return rc;
    }
    return VO_OK;
}

// BGR staging -> the 2 * n_seq raw gray planes of `slot` (cv::cvtColor(BGR2GRAY) of utils.cpp:179,189)
static int convert_pairs(vo_ctx* ctx, int slot)
{
    const int w = ctx->w, h = ctx->h, n = ctx->seq_n;
    ctx->launches += vo_launch_bgr_to_gray(nullptr, vo_packed_bgr(ctx->d_bgr, w), (size_t)3 * w * h, ctx->d_raw + (size_t)(2 * n * slot) * w * h,
                                           (size_t)w * h, w, h, 2 * n, ctx->stream, ctx->seq_sized ? ctx->d_geo + 2 * n * slot : nullptr);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

// the glue kernels' arguments for the n_seq units of buffer parity p (units u0 .. u0 + n_seq - 1); s0 = the image slot of
// the frame's previous pairs, whose geometry entries give each sequence's bucket grid
static void seq_args(vo_ctx* ctx, int p, SeqArgs& a, int s0 = 0)
{
    memset(&a, 0, sizeof(a));
    const int n = ctx->seq_n, u0 = p * n;
    const size_t uo = (size_t)u0 * ctx->cap, cs = (size_t)ctx->units * ctx->cap;
    a.corners = ctx->d_corners + (size_t)u0 * ctx->corner_cap; a.n_det = ctx->d_ndet + u0; a.corner_cap = ctx->corner_cap;
    a.feat_pts = ctx->d_feat_pts; a.feat_ages = ctx->d_feat_ages; a.cnt = ctx->d_feat_cnt; a.feat_cap = ctx->feat_cap;
    // each sequence's refill threshold and bucketing (visualOdometry.cpp:95,106-107, bucket.cpp:16 at the defaults)
    a.par = ctx->d_par + u0;
    a.rows = ctx->h; a.cols = ctx->w;
    // sequence q: plane 2q of image slot s0 (a started sequence's size reaches the three slots one staged pair at a time)
    a.geo = ctx->seq_sized ? ctx->d_geo + 2 * n * s0 : nullptr; a.geo_stride = 2;
    a.bucket = ctx->d_bucket; a.bucket_cap = ctx->bucket_cap;
    a.out_pts = ctx->d_pts_in + uo; a.out_ages = ctx->d_ages_in + uo; a.out_n = ctx->d_npts + u0; a.out_cap = ctx->cap;
    a.valid_l1 = ctx->d_valid4 + 2 * cs + uo; a.n5 = ctx->d_n5 + u0; a.ages_out = ctx->d_ages_out + uo; a.n3 = ctx->d_n3 + u0;
    a.res = ctx->d_results + u0;
    a.tprev = ctx->d_tprev + 3 * (size_t)((1 - p) * n);     // the next frame solves from this frame's translation
    a.tprev_cur = ctx->d_tprev + 3 * (size_t)u0;
    a.err = ctx->d_seq_err + 1 + u0; a.err_out = ctx->d_seq_err + 1 + u0;      // one word per unit = per sequence and frame in flight
    a.live = ctx->d_seq_live + u0;
}

// bucketingFeatures() reads back (rows/bs + 1) x (cols/bs + 1) buckets of features_per_bucket slots at most
// (feature.cpp:242-249), bs = rows / bucket_rows_divisor, at a sequence's parameters p: the bound of every per-frame
// point count (the largest over the sequences' sizes and parameters).  In 64 bits, so that no features_per_bucket
// overflows it; the begin and start calls keep it within max_features.
static long long seq_grid(const vo_params& p, int w, int h)
{
    const int d = p.bucket_rows_divisor, bs = h / d > 0 ? h / d : 1;
    return (long long)(h / bs + 1) * (w / bs + 1) * p.features_per_bucket;
}
static long long seq_grid(const vo_ctx* ctx)
{
    long long g = 0;
    for (int q = 0; q < ctx->seq_n; q++) g = std::max(g, seq_grid(ctx->seq_par[q], ctx->seq_w[q], ctx->seq_h[q]));
    return g;
}

// the bucketing checks of a w x h sequence at parameters p (who_q: "sequence 3", "slot 3", "the envelope"): a zero bucket
// size is refused (VO_E_UNSUPPORTED, as images under 10 rows always were: the reference divides by zero), and so is a
// bound above the per-unit capacity (VO_E_CAPACITY: the point lists of every stage after the bucketing hold max_features
// points)
static int seq_grid_check(vo_ctx* ctx, const char* who, const char* who_q, int w, int h, const vo_params& p)
{
    if (h / p.bucket_rows_divisor <= 0) {
        vo_set_error(ctx, "%s: %s: %d x %d is too small for the rows/%d bucket size", who, who_q, w, h, p.bucket_rows_divisor);
        return VO_E_UNSUPPORTED;
    }
    const long long g = seq_grid(p, w, h);
    if (g > ctx->cap) {
        vo_set_error(ctx, "%s: %s: %d x %d reads back up to %lld points at features_per_bucket = %d (bucket size rows / %d), "
                          "above max_features = %d", who, who_q, w, h, g, p.features_per_bucket, p.bucket_rows_divisor,
                     ctx->cap);
        return VO_E_CAPACITY;
    }
    return VO_OK;
}

// the mono branch of buffer units unit .. unit + n_prob - 1 (one problem each): pointsLeft_t0 / pointsLeft_t1 = the
// filtered L0 / L1 lists (d_valid4 planes 0, 2), scratch block u for unit u
static void seq_ess_args(vo_ctx* ctx, int unit, int n_prob, EssArgs& a)
{
    memset(&a, 0, sizeof(a));
    const size_t uo = (size_t)unit * ctx->cap, cs = (size_t)ctx->units * ctx->cap;
    vo_ess_bind(a, (uint8_t*)ctx->d_seq_ess + (size_t)unit * ctx->seq_ess_bytes, ctx->seq_ess_cap, VO_ESS_ITERS);
    a.n = ctx->d_n5 + unit;
    a.cal = ctx->d_cal + unit;                                // focal / pp / threshold of each unit's P_l
    a.pts0 = ctx->d_valid4 + uo; a.pts1 = ctx->d_valid4 + 2 * cs + uo;
    a.n_prob = n_prob;
    a.scratch_stride = a.result_stride = ctx->seq_ess_bytes; a.pts_stride = ctx->cap; a.n_stride = 1; a.cal_stride = 1;
}

// per-unit scratch of the mono branch for the 2 * n units of n sequences, sized for the bucket grid (outside any capture:
// the begin calls)
static int seq_mono_scratch(vo_ctx* ctx, int n)
{
    const long long grid = seq_grid(ctx);
    const int n_max = (int)std::min<long long>(grid, ctx->cap);
    if (!ctx->seq_mono_stream) {
        VO_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->seq_mono_stream, cudaStreamNonBlocking));
        for (int k = 0; k < 2; k++) VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->seq_mono_ev[k], cudaEventDisableTiming));
    }
    if (ctx->d_seq_ess && ctx->seq_ess_cap >= n_max && ctx->seq_ess_units >= 2 * n) return VO_OK;
    vo_drop_graphs(ctx);                                      // captured graphs hold the old blocks
    if (ctx->d_seq_ess) { VO_CUDA_CHECK(cudaDeviceSynchronize()); cudaFree(ctx->d_seq_ess); ctx->d_seq_ess = nullptr; ctx->seq_ess_units = 0; }
    const size_t bytes = (vo_ess_scratch_bytes(n_max, VO_ESS_ITERS) + 255) / 256 * 256;
    VO_CUDA_CHECK(cudaMalloc(&ctx->d_seq_ess, 2 * (size_t)n * bytes));
    ctx->seq_ess_bytes = bytes; ctx->seq_ess_cap = n_max; ctx->seq_ess_units = 2 * n;
    return VO_OK;
}

// front stage of one frame of every sequence on the caller's stream; s0 / s1 = image slots of the previous / new pairs,
// p = buffer parity (per-frame buffers: units p * n_seq .. p * n_seq + n_seq - 1)
static int seq_front(vo_ctx* ctx, int s0, int s1, int p, bool bgr)
{
    const int n = ctx->seq_n, unit = p * n;
    const int L0 = 2 * n * s0, R0 = L0 + 1, L1 = 2 * n * s1, R1 = L1 + 1;
    // image planes are addressed from plane 0 whatever the parity; sequence q's pair of a slot is planes 2q, 2q + 1 of it
    const View v{unit, n, ctx->stream, 0, 2, ctx->seq_lk_bound, ctx->seq_sized};
    int rc;
    if (bgr && (rc = convert_pairs(ctx, s1))) return rc;
    // the new pairs' pyramids (the previous pairs' are already resident)
    if ((rc = vo_run_pyramid(ctx, L1, 2 * n, ctx->stream, ctx->seq_sized))) return rc;
    // matchingFeatures(): FAST refill on the t0 left image -> bucketing -> circular matching -> filters
    if ((rc = vo_run_fast(ctx, v, L0, false, ctx->d_par))) return rc;
    SeqArgs a;
    seq_args(ctx, p, a, s0);
    ctx->launches += vo_launch_seq_append(a, n, ctx->stream);
    ctx->launches += vo_launch_seq_bucket(a, n, ctx->stream);
    const int ip[4] = {L0, R0, R1, L1}, in[4] = {R0, R1, L1, L0};
    if ((rc = vo_run_lk_ring(ctx, v, 4, ip, in, false, ctx->d_par))) return rc;
    if ((rc = vo_run_filter(ctx, v, true, ctx->d_par))) return rc;
    if (ctx->seq_mono) {        // findEssentialMat + recoverPose on (L0, L1) of every sequence, beside the carry and the triangulation
        EssArgs e;
        seq_ess_args(ctx, unit, n, e);
        VO_CUDA_CHECK(cudaEventRecord(ctx->seq_mono_ev[0], ctx->stream));
        VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->seq_mono_stream, ctx->seq_mono_ev[0], 0));
        ctx->launches += vo_launch_essential(e, ctx->seq_mono_stream);
        VO_CUDA_CHECK(cudaGetLastError());
        VO_CUDA_CHECK(cudaEventRecord(ctx->seq_mono_ev[1], ctx->seq_mono_stream));
    }
    // state carry: features.points = pointsLeft_t1, ages keep their A3 length
    ctx->launches += vo_launch_seq_carry(a, n, ctx->stream);
    const size_t cs = (size_t)ctx->units * ctx->cap;
    if ((rc = vo_run_triangulate(ctx, v, ctx->d_valid4, ctx->d_valid4 + cs, ctx->d_n5, ctx->d_cal))) return rc;
    if (ctx->seq_mono) VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->seq_mono_ev[1], 0));
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

// back stage on side stream 0: trackingFrame2Frame's PnP + translation carry (+ the mono rotation into the record)
static int seq_back(vo_ctx* ctx, int p)
{
    cudaStream_t st = ctx->lane[0].side;
    const int n = ctx->seq_n, unit = p * n;
    const View v{unit, n, st, 0};
    const size_t cs = (size_t)ctx->units * ctx->cap;
    int rc;
    if ((rc = vo_run_pnp(ctx, v, ctx->d_valid4 + 2 * cs, ctx->d_n5, ctx->d_cal, ctx->d_par))) return rc;
    SeqArgs a;
    seq_args(ctx, p, a);
    ctx->launches += vo_launch_seq_finish(a, n, st);
    if (ctx->seq_mono) {
        EssArgs e;
        seq_ess_args(ctx, unit, n, e);
        ctx->launches += vo_launch_seq_mono(a, e.result, e.result_stride, n, st);
    }
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

// pinned staging of the sequence mode: the records and error words of the 2 * n_seq units (both parities) |
// EssResult[2 * n_seq] (mono sequences only) | vo_dimage[6 * n_seq] (device-image descriptors, one per raw plane of the
// three-slot ring, indexed by plane: entry 2 * n_seq * s + 2q + k is sequence q's image k of slot s).  Slot s's entries are
// rewritten by the submission that stages into s, three submissions after the one that last copied them to the device;
// with at most two submissions in flight that one has been waited for, so its copy has run -- when the wait blocks.
// vo_mseq_wait_device does not, so runs begun with VO_MSEQ_DEVICE_RESULTS wait for seq_tab_ev[s], recorded after the copy.
struct SeqPinned { vo_unit_result_dev* rec; int* err; EssResult* ess; vo_dimage* tab; size_t bytes; };
static SeqPinned seq_pinned(vo_ctx* ctx, int n)
{
    auto up = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t o_err = up(2 * (size_t)n * sizeof(vo_unit_result_dev)), o_ess = up(o_err + 2 * (size_t)n * sizeof(int));
    const size_t o_tab = up(o_ess + 2 * (size_t)n * sizeof(EssResult)), end = up(o_tab + 6 * (size_t)n * sizeof(vo_dimage));
    uint8_t* b = (uint8_t*)ctx->h_pinned;
    return SeqPinned{(vo_unit_result_dev*)b, (int*)(b + o_err), (EssResult*)(b + o_ess), (vo_dimage*)(b + o_tab), end};
}

// the per-sequence device state (FeatureSet, bucket scratch, error and live words) for n sequences, in one allocation that
// lives until the batch state is re-allocated (outside any capture: vo_seq_begin / vo_mseq_begin)
static int seq_state_alloc(vo_ctx* ctx, int n)
{
    if (ctx->d_seq_state && ctx->seq_n_cap >= n) return VO_OK;
    vo_drop_graphs(ctx);                                      // captured graphs hold the old blocks
    if (ctx->d_seq_state) { VO_CUDA_CHECK(cudaDeviceSynchronize()); cudaFree(ctx->d_seq_state); ctx->d_seq_state = nullptr; ctx->seq_n_cap = 0; }
    auto up = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t fc = (size_t)n * ctx->feat_cap;
    const size_t o_ages = up(fc * sizeof(float2)), o_cnt = up(o_ages + fc * sizeof(int)), o_bucket = up(o_cnt + 2 * (size_t)n * sizeof(int));
    const size_t o_err = up(o_bucket + (size_t)n * ctx->bucket_cap * sizeof(int)), o_live = up(o_err + (1 + 2 * (size_t)n) * sizeof(int));
    const size_t bytes = up(o_live + 2 * (size_t)n * sizeof(int));
    VO_CUDA_CHECK(cudaMalloc(&ctx->d_seq_state, bytes));
    uint8_t* b = (uint8_t*)ctx->d_seq_state;
    ctx->d_feat_pts = (float2*)b; ctx->d_feat_ages = (int*)(b + o_ages); ctx->d_feat_cnt = (int*)(b + o_cnt);
    ctx->d_bucket = (int*)(b + o_bucket); ctx->d_seq_err = (int*)(b + o_err); ctx->d_seq_live = (int*)(b + o_live);
    ctx->seq_n_cap = n;
    return VO_OK;
}

static int seq_events(vo_ctx* ctx)
{
    if (!ctx->seq_front_ev[0])
        for (int k = 0; k < 2; k++) {
            VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->seq_front_ev[k], cudaEventDisableTiming));
            VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->seq_back_ev[k], cudaEventDisableTiming));
        }
    return vo_ensure_lanes(ctx);
}

// retire every frame in flight without reporting it (state queries / re-begin / destroy)
static int seq_drain(vo_ctx* ctx)
{
    if (ctx->seq_inflight > 0) {
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->lane[0].side));
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    }
    return VO_OK;
}

// where the new pairs of a begin or submit call come from: host images (gray or BGR, sequence q's pitch[q] bytes per row)
// or device images (vo_seq_*_device, vo_mseq_*_device: sequence q's pair is dl[q] / dr[q]).  In a multi-sequence
// submission a NULL pair (host pointers, or descriptors whose data are NULL) retires its sequence.
struct SeqPairs {
    const uint8_t* const* lefts; const uint8_t* const* rights; const size_t* pitch; int channels;
    bool device; const vo_dimage* dl; const vo_dimage* dr;
    bool bgr() const { return !device && channels == 3; }
    bool left(int q) const { return device ? dl[q].data != nullptr : lefts[q] != nullptr; }
    bool right(int q) const { return device ? dr[q].data != nullptr : rights[q] != nullptr; }
};
static SeqPairs host_pairs(const uint8_t* const* lefts, const uint8_t* const* rights, const size_t* pitch, int channels)
{
    return SeqPairs{lefts, rights, pitch, channels, false, nullptr, nullptr};
}
static SeqPairs device_pairs(const vo_dimage* lefts, const vo_dimage* rights) { return SeqPairs{nullptr, nullptr, nullptr, 1, true, lefts, rights}; }

// the new pairs' own checks (w[q]: sequence q's image width; begin: the first pairs, which every sequence needs; starting[q]:
// the pair starts a new sequence in slot q of a running submission, so it needs both images and may follow a retirement).
// A pitch is checked only where a pair is read: a retiring sequence's is not.
static int seq_pairs_check(vo_ctx* ctx, const char* who, bool multi, int n, const int* w, const SeqPairs& in, bool begin,
                           const char* starting = nullptr)
{
    int rc;
    if (in.device) {
        if (!in.dl || !in.dr) { vo_set_error(ctx, "%s: bad argument", who); return VO_E_INVALID; }
        // a single sequence's images, and every image of a pair that is read, as sequence q's w[q] pixels
        char name[32];
        for (int q = 0; q < n; q++)
            for (int k = 0; k < 2; k++) {
                const vo_dimage* im = k ? in.dr + q : in.dl + q;
                if (multi && !in.left(q) && !in.right(q)) continue;
                if (multi && !im->data) continue;             // one image of a pair: refused below
                snprintf(name, sizeof(name), multi ? "%s%c[%d]" : "%s%c", k ? "right" : "left", begin ? '0' : '1', q);
                if ((rc = vo_check_dimage(ctx, who, name, im, w[q]))) return rc;
            }
    } else {
        if (in.channels != 1 && in.channels != 3) { vo_set_error(ctx, "%s: channels must be 1 (gray) or 3 (BGR)", who); return VO_E_INVALID; }
        if (!in.lefts || !in.rights || !in.pitch || (!multi && (!in.lefts[0] || !in.rights[0]))) {
            vo_set_error(ctx, "%s: bad argument", who);
            return VO_E_INVALID;
        }
        for (int q = 0; q < n; q++)
            if (in.lefts[q] && in.pitch[q] < (size_t)w[q] * in.channels) {
                vo_set_error(ctx, "%s: bad argument (sequence %d: pitch %zu < %d pixels x %d channel(s))", who, q, in.pitch[q], w[q], in.channels);
                return VO_E_INVALID;
            }
    }
    for (int q = 0; multi && q < n; q++) {
        const bool l = in.left(q), r = in.right(q);
        const bool first = begin || (starting && starting[q]);
        if (first && !(l && r)) { vo_set_error(ctx, "%s: sequence %d has no first pair", who, q); return VO_E_INVALID; }
        if (!begin && l != r) { vo_set_error(ctx, "%s: sequence %d has only one image (a NULL pair retires it)", who, q); return VO_E_INVALID; }
        if (!first && l && ctx->seq_retired[q]) { vo_set_error(ctx, "%s: sequence %d was retired", who, q); return VO_E_INVALID; }
    }
    return VO_OK;
}

// the new pairs into image slot `slot` on st: host pairs as upload_pairs writes them; device pairs converted into the
// slot's 2 * n_seq raw planes by ONE k_bgr_to_gray launch through the slot's entries of the pinned descriptor table (a
// retiring or empty slot's entries have data == NULL: its planes keep their stale contents, as a skipped host upload
// leaves them), each image at its plane's own size from the geometry table in a run of several sizes
static int stage_pairs(vo_ctx* ctx, int slot, const SeqPairs& in, cudaStream_t st)
{
    if (!in.device) return upload_pairs(ctx, slot, in.lefts, in.rights, in.pitch, in.channels, st);
    const int n = ctx->seq_n;
    vo_dimage* tab = seq_pinned(ctx, n).tab + 2 * n * slot;
    if (ctx->seq_dres) VO_CUDA_CHECK(cudaEventSynchronize(ctx->seq_tab_ev[slot]));
    for (int q = 0; q < n; q++) { tab[2 * q] = in.dl[q]; tab[2 * q + 1] = in.dr[q]; }
    const int rc = vo_ingest_device(ctx, tab, 2 * n, 2 * n * slot, st, ctx->seq_sized ? ctx->d_geo + 2 * n * slot : nullptr);
    if (!rc && ctx->seq_dres) VO_CUDA_CHECK(cudaEventRecord(ctx->seq_tab_ev[slot], st));
    return rc;
}

// n new sequences (multi: begun by vo_mseq_begin*) from their first pairs `in`; sequence q is w[q] x h[q] and runs with
// the matrices P_l + 12q / P_r + 12q; every frame also runs the mono_rotation branch with the option "mono_rotation"
// (vo_seq_begin*) or the flag VO_MSEQ_MONO_ROTATION (vo_mseq_begin_ex / _calib / _sized).  Refused, before anything
// changes, while a batch submission has not been waited for: it still uses the unit buffers and the pinned block.  A
// running sequence mode of the same kind is drained and ended; one of the other kind only when it is idle.
// in == nullptr (vo_mseq_open): n empty slots at the envelope w[q] x h[q] (one value repeated), no matrices, no pairs; the
// run reads the geometry table whatever sizes its sequences get.
static int seq_begin(vo_ctx* ctx, const char* who, bool multi, int n, int flags, const int* w, const int* h, const float* P_l,
                     const float* P_r, const SeqPairs* in)
{
    if (!ctx) return VO_E_INVALID;
    const bool open = in == nullptr;
    if (multi) {
        const int known = VO_MSEQ_MONO_ROTATION | VO_MSEQ_DEVICE_RESULTS;
        if (flags & ~known) { vo_set_error(ctx, "%s: unknown flag bits 0x%x", who, (unsigned)(flags & ~known)); return VO_E_INVALID; }
        if (n < 1) { vo_set_error(ctx, "%s: n_seq = %d, need at least one sequence", who, n); return VO_E_INVALID; }
        if (n > VO_MSEQ_MAX) {
            vo_set_error(ctx, "%s: %s = %d, a context holds at most %d sequences", who, open ? "n_slots" : "n_seq", n, VO_MSEQ_MAX);
            return open ? VO_E_INVALID : VO_E_CAPACITY;
        }
    }
    if ((!open && (!P_l || !P_r)) || !w || !h) { vo_set_error(ctx, "%s: bad argument", who); return VO_E_INVALID; }
    for (int q = 0; q < n; q++)
        if (w[q] <= 0 || h[q] <= 0) { vo_set_error(ctx, "%s: bad argument (sequence %d is %d x %d)", who, q, w[q], h[q]); return VO_E_INVALID; }
    int rc;
    if (!open && (rc = seq_pairs_check(ctx, who, multi, n, w, *in, true))) return rc;
    // each sequence's parameters: its slot's setting (vo_mseq_params), the context's for vo_seq_*
    const std::vector<vo_params> par = multi ? std::vector<vo_params>(ctx->slot_par.begin(), ctx->slot_par.begin() + n)
                                             : std::vector<vo_params>(1, ctx->p);
    // the envelope of the sizes (the planes' allocation) and the one pyramid depth they must share
    int W = 0, H = 0;
    const int depth = vo_pyr_depth(w[0], h[0], ctx->p.lk_max_level);
    for (int q = 0; q < n; q++) {
        char who_q[32];
        snprintf(who_q, sizeof(who_q), open ? "the envelope at slot %d's parameters" : "sequence %d", q);
        if ((rc = seq_grid_check(ctx, who, who_q, w[q], h[q], par[q]))) return rc;
        if (vo_pyr_depth(w[q], h[q], ctx->p.lk_max_level) != depth) {
            vo_set_error(ctx, "%s: sequence 0 (%d x %d) has %d pyramid levels, sequence %d (%d x %d) %d: one run needs one pyramid depth",
                         who, w[0], h[0], depth, q, w[q], h[q], vo_pyr_depth(w[q], h[q], ctx->p.lk_max_level));
            return VO_E_UNSUPPORTED;
        }
        W = std::max(W, w[q]); H = std::max(H, h[q]);
    }
    bool sized = open;
    for (int q = 0; q < n; q++) sized = sized || w[q] != W || h[q] != H;
    // the mono_rotation branch of several sequences is asked for with the flag only: the context option, which
    // vo_seq_begin* take, would otherwise silently pick (or drop) the branch for a whole set of sequences
    if (multi && ctx->mono_opt) {
        vo_set_error(ctx, "%s: the option \"mono_rotation\" is not supported with several sequences (use the flag "
                          "VO_MSEQ_MONO_ROTATION of vo_mseq_begin_ex)", who);
        return VO_E_UNSUPPORTED;
    }
    if ((rc = vo_refuse_pending_batches(ctx, who))) return rc;
    if (ctx->seq_active && ctx->seq_multi != multi && ctx->seq_inflight > 0) {
        vo_set_error(ctx, "%s: %d frame(s) submitted with %s have not been waited for", who, ctx->seq_inflight,
                     multi ? "vo_seq_submit" : "vo_mseq_submit");
        return VO_E_INVALID;
    }
    const bool mono = multi ? (flags & VO_MSEQ_MONO_ROTATION) != 0 : ctx->mono_opt;
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    if (ctx->seq_active && (rc = seq_drain(ctx))) return rc;
    ctx->seq_inflight = 0;
    ctx->seq_active = false;
    // two per-frame buffer units per sequence (frames in flight)
    if ((rc = vo_ensure_state(ctx, W, H, 2 * n, depth))) return rc;
    if ((rc = seq_state_alloc(ctx, n))) return rc;
    if ((rc = seq_events(ctx))) return rc;
    // the frame graphs are captured for one sequence count, with or without the mono branch (which a sequence keeps),
    // and with or without the geometry table (not for the sizes in it)
    if (ctx->seq_n != n) { vo_drop_graphs(ctx); ctx->seq_n = n; }
    ctx->seq_multi = multi;
    if (ctx->seq_mono != mono) { vo_drop_graphs(ctx); ctx->seq_mono = mono; }
    if (ctx->seq_sized != sized) { vo_drop_graphs(ctx); ctx->seq_sized = sized; }
    ctx->seq_w.assign(w, w + n);
    ctx->seq_h.assign(h, h + n);
    ctx->seq_par = par;
    if (sized) {        // sequence q's planes 2q, 2q + 1 of each of the three image slots
        std::vector<PlaneGeom> g(6 * (size_t)n);
        for (int s = 0; s < 3; s++)
            for (int q = 0; q < n; q++) g[2 * n * s + 2 * q] = g[2 * n * s + 2 * q + 1] = vo_plane_geom(ctx, w[q], h[q]);
        if ((rc = vo_write_geo(ctx, 0, 6 * n, g.data()))) return rc;
    }
    // the LK launch bound (and the mono scratch): the begun sizes' largest bucket grid, or the envelope's for an open run
    ctx->seq_lk_bound = (int)seq_grid(ctx);
    if (ctx->seq_mono && (rc = seq_mono_scratch(ctx, n))) return rc;
    if ((rc = vo_ensure_pinned(ctx, seq_pinned(ctx, n).bytes))) return rc;
    ctx->seq_dres = multi && (flags & VO_MSEQ_DEVICE_RESULTS);
    if (ctx->seq_dres && !ctx->d_seq_pose) {
        VO_CUDA_CHECK(cudaMalloc(&ctx->d_seq_pose, 16 * (size_t)VO_MSEQ_MAX * sizeof(double)));
        for (int s = 0; s < 3; s++) VO_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->seq_tab_ev[s], cudaEventDisableTiming));
    }
    // sequence q owns the buffer units q and n + q (both parities): both entries carry its camera and its parameters (a
    // start writes them)
    if (!open && (rc = vo_set_calibration(ctx, 0, 2 * n, P_l, P_r, n))) return rc;
    {
        std::vector<UnitParams> e(2 * (size_t)n);
        for (int u = 0; u < 2 * n; u++) e[u] = vo_unit_params(par[u % n]);
        if ((rc = vo_write_params(ctx, 0, 2 * n, e.data()))) return rc;
    }
    ctx->seq_slot = 0;
    ctx->seq_submitted = 0;
    ctx->seq_pose.assign(16 * (size_t)n, 0.0);
    for (int q = 0; q < n; q++)
        for (int i = 0; i < 4; i++) ctx->seq_pose[16 * q + 5 * i] = 1.0;
    // (a pageable copy: the host vector may go once the call returns, which the synchronise below covers anyway)
    if (ctx->seq_dres)
        VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_seq_pose, ctx->seq_pose.data(), 16 * (size_t)n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    ctx->seq_retired.assign(n, open ? 1 : 0);
    ctx->seq_live.assign(2 * (size_t)n, open ? 0 : 1);
    ctx->seq_cal_next.assign(2 * (size_t)n, CamCalib{});
    ctx->seq_par_next.assign(2 * (size_t)n, UnitParams{});
    ctx->seq_cal_due.assign(2 * (size_t)n, 0);
    ctx->seq_geo_due.assign(n, 0);
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_feat_cnt, 0, 2 * (size_t)n * sizeof(int), ctx->stream));
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_seq_err, 0, (1 + 2 * (size_t)n) * sizeof(int), ctx->stream));
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_seq_live, open ? 0 : 1, 2 * (size_t)n * sizeof(int), ctx->stream));   // any non-zero word is live
    VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_tprev, 0, 6 * (size_t)n * sizeof(double), ctx->stream));   // translation = zeros (main.cpp:82)
    // the first pairs into image slot 0 on the caller's stream, after the work already enqueued there (the synchronise
    // below is the release of device images)
    if (!open) {
        if ((rc = stage_pairs(ctx, 0, *in, ctx->stream)) || (in->bgr() && (rc = convert_pairs(ctx, 0)))) return rc;
        if ((rc = vo_run_pyramid(ctx, 0, 2 * n, ctx->stream, sized))) return rc;
    }
    // both event pairs start out signalled, so the first two frames do not wait for a predecessor
    for (int k = 0; k < 2; k++) {
        VO_CUDA_CHECK(cudaEventRecord(ctx->seq_front_ev[k], ctx->stream));
        VO_CUDA_CHECK(cudaEventRecord(ctx->seq_back_ev[k], ctx->stream));
    }
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->seq_active = true;
    return VO_OK;
}

enum SeqCall { SEQ_SUBMIT, SEQ_WAIT, SEQ_QUERY };

// the checks every frame call starts with: the sequences run, begun by this mode (multi: vo_mseq_begin*; the frame calls
// of one mode are refused while the other one runs), and the frames in flight allow the call (a submission: fewer than
// two; a wait: at least one)
static int seq_frame_check(vo_ctx* ctx, const char* who, bool multi, SeqCall call)
{
    const char* begin = multi ? "vo_mseq_begin" : "vo_seq_begin";
    if (ctx->seq_active && ctx->seq_multi != multi) {
        vo_set_error(ctx, "%s: the running sequences were begun with %s", who, multi ? "vo_seq_begin" : "vo_mseq_begin");
        return VO_E_INVALID;
    }
    if (!ctx->seq_active) {
        vo_set_error(ctx, call == SEQ_WAIT ? "%s: no frame in flight; call %s first" : "%s: call %s first", who, begin);
        return VO_E_INVALID;
    }
    if (call == SEQ_WAIT && ctx->seq_inflight <= 0) { vo_set_error(ctx, "%s: no frame in flight", who); return VO_E_INVALID; }
    if (call == SEQ_SUBMIT && ctx->seq_inflight >= 2) {
        vo_set_error(ctx, "%s: two frames are in flight already; call %s", who, multi ? "vo_mseq_wait" : "vo_seq_wait");
        return VO_E_INVALID;
    }
    return VO_OK;
}

// One frame of every sequence (a NULL pair retires its sequence): the new pairs into the image slot s1 that neither the
// running nor the previous frame reads, the front stage (gray frames replay the gray graph whatever their source), the
// back stage, the record copies
// The checks of a submission's starts (vo_mseq_submit_start), before anything changes: starting[q] marks slot q's pair as
// the first pair of a new sequence, w[q] is then its width (for the pitch check).
static int seq_starts_check(vo_ctx* ctx, const char* who, int n_start, const vo_mseq_start* starts, std::vector<char>& starting,
                            std::vector<int>& w)
{
    const int n = ctx->seq_n;
    if (n_start < 0 || (n_start > 0 && !starts)) { vo_set_error(ctx, "%s: bad argument (n_start = %d)", who, n_start); return VO_E_INVALID; }
    for (int i = 0; i < n_start; i++) {
        const vo_mseq_start& s = starts[i];
        if (s.slot < 0 || s.slot >= n) { vo_set_error(ctx, "%s: start %d: slot %d of %d", who, i, s.slot, n); return VO_E_INVALID; }
        if (starting[s.slot]) { vo_set_error(ctx, "%s: start %d: slot %d is started twice", who, i, s.slot); return VO_E_INVALID; }
        if (s.w <= 0 || s.h <= 0) { vo_set_error(ctx, "%s: start %d: bad size %d x %d", who, i, s.w, s.h); return VO_E_INVALID; }
        starting[s.slot] = 1;
        w[s.slot] = s.w;
    }
    return VO_OK;
}

// the sizes a run can start: the run's planes, pyramid depth and mono scratch are those of its begin; the bucketing
// scratch holds any bucket bound within max_features
static int seq_starts_fit(vo_ctx* ctx, const char* who, int n_start, const vo_mseq_start* starts)
{
    for (int i = 0; i < n_start; i++) {
        const int w = starts[i].w, h = starts[i].h, q = starts[i].slot;
        if (!ctx->seq_sized && (w != ctx->w || h != ctx->h)) {
            vo_set_error(ctx, "%s: slot %d: %d x %d in a run of the one size %d x %d (a run begun with vo_mseq_open or "
                              "vo_mseq_begin_sized starts other sizes)", who, q, w, h, ctx->w, ctx->h);
            return VO_E_UNSUPPORTED;
        }
        if (w > ctx->w || h > ctx->h) {
            vo_set_error(ctx, "%s: slot %d: %d x %d is outside the run's envelope %d x %d", who, q, w, h, ctx->w, ctx->h);
            return VO_E_UNSUPPORTED;
        }
        char who_q[32];
        snprintf(who_q, sizeof(who_q), "slot %d", q);
        int rc;
        if ((rc = seq_grid_check(ctx, who, who_q, w, h, ctx->slot_par[q]))) return rc;
        const int depth = vo_pyr_depth(w, h, ctx->p.lk_max_level);
        if (depth != ctx->pg.nlevels) {
            vo_set_error(ctx, "%s: slot %d: %d x %d has %d pyramid levels, the run %d", who, q, w, h, depth, ctx->pg.nlevels);
            return VO_E_UNSUPPORTED;
        }
        const int grid = (int)seq_grid(ctx->slot_par[q], w, h);
        if (ctx->seq_mono && std::min(grid, ctx->cap) > ctx->seq_ess_cap) {
            vo_set_error(ctx, "%s: slot %d: %d x %d needs mono scratch for %d points, the run reserved %d", who, q, w, h,
                         std::min(grid, ctx->cap), ctx->seq_ess_cap);
            return VO_E_CAPACITY;
        }
    }
    return VO_OK;
}

// One frame of every sequence (a NULL pair retires its sequence; starts: the listed slots' pairs begin new sequences,
// vo_mseq_submit_start): the new pairs into the image slot s1 that neither the running nor the previous frame reads, the
// front stage (gray frames replay the gray graph whatever their source), the back stage, the record copies.
//
// A start in slot q at submission k (parity p) resets the slot's state against the two frames that may be in flight:
//   live word      unit p * n + q is 0 in frame k (its stages skip the slot, as for a retired one; the wait reports
//                  VO_MSEQ_STARTED from the host copy) and 1 from frame k + 1 on.  Like a retirement, a unit's word is
//                  written by the next submission of its parity, after the back stage that last read it.
//   FeatureSet     d_feat_cnt of q zeroed on the front stream: after the carry of frame k - 1 (stream order), and frame k
//                  skips the slot, so frame k + 1 refills from FAST on the first pair as vo_seq_begin's first push does.
//   translation    the back stage of frame k - 1 (side stream) writes tprev[p n + q], and k_seq_finish of frame k copies
//                  it into tprev[(1 - p) n + q] for the skipped slot: the zeroing goes on the side stream right after the
//                  back stage of frame k, so frame k + 1 solves from zeros (main.cpp:82).
//   calibration    (and the parameter entry, the slot's vo_mseq_params setting: the same two writes) unit p n + q was
//                  last read by frame k - 2 (the front stream has waited for its back stage): written now.  Unit
//                  (1 - p) n + q may still be read by the kernels of frame k - 1: written by submission k + 1, after
//                  seq_back_ev[1 - p].
//   geometry       the entries of q's planes in image slot s are written when a pair of the new sequence is staged into
//                  s (s1 of frames k, k + 1, k + 2): s1 was last read by frame k - 2, and slot s0 of frame k is still being
//                  written by the pyramid launch of frame k - 1.
//   frame_pose     reset by the wait of frame k: the waits of frames k - 2 and k - 1 still integrate the old sequence.
static int seq_submit(vo_ctx* ctx, const char* who, bool multi, const SeqPairs& in, int n_start = 0, const vo_mseq_start* starts = nullptr)
{
    if (!ctx) return VO_E_INVALID;
    int rc;
    if ((rc = seq_frame_check(ctx, who, multi, SEQ_SUBMIT))) return rc;
    if (ctx->seq_dres && !in.device) {
        vo_set_error(ctx, "%s: the sequences were begun with VO_MSEQ_DEVICE_RESULTS, which takes frames through "
                          "vo_mseq_submit_device only (a wait that does not block cannot release host images)", who);
        return VO_E_INVALID;
    }
    const int n = ctx->seq_n;
    // a submission without starts checks its pairs against the running sizes, with no per-slot copies
    std::vector<char> starting;
    std::vector<int> wq;
    const int* w = ctx->seq_w.data();
    const char* st = nullptr;
    if (n_start || starts) {
        starting.assign(n, 0);
        wq = ctx->seq_w;
        if ((rc = seq_starts_check(ctx, who, n_start, starts, starting, wq))) return rc;
        w = wq.data(); st = starting.data();
    }
    if ((rc = seq_pairs_check(ctx, who, multi, n, w, in, false, st)) ||
        (rc = seq_starts_fit(ctx, who, n_start, starts)))
        return rc;
    for (int q = 0; multi && q < n; q++)
        if (!in.left(q)) ctx->seq_retired[q] = 1;
    for (int i = 0; i < n_start; i++) {
        const vo_mseq_start& s = starts[i];
        ctx->seq_retired[s.slot] = 0;
        ctx->seq_w[s.slot] = s.w; ctx->seq_h[s.slot] = s.h;
        ctx->seq_par[s.slot] = ctx->slot_par[s.slot];
        ctx->seq_geo_due[s.slot] = 3;
        // a larger bucket grid is a front graph of its own; the bound never shrinks within a run
        ctx->seq_lk_bound = std::max(ctx->seq_lk_bound, (int)seq_grid(ctx->seq_par[s.slot], s.w, s.h));
    }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const int p = (int)(ctx->seq_submitted & 1);
    const int s0 = ctx->seq_slot, s1 = (s0 + 1) % 3;
    const bool bgr = in.bgr();
    // Producer ordering of device images: the conversion reads them after the caller's work enqueued so far.  The event is
    // recorded BEFORE the front stream waits for frame k-2's back stage below, so that the conversion does not queue
    // behind that pose solve.
    if (in.device) VO_CUDA_CHECK(cudaEventRecord(ctx->fork_ev, ctx->stream));
    // the per-frame buffers of parity p were last read by the back stage of frame k-2
    VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->seq_back_ev[p], 0));
    // calibration and parameter entries of parity p deferred by a start in the previous submission, then this
    // submission's starts
    for (int q = 0; q < n; q++)
        if (ctx->seq_cal_due[p * n + q]) {
            if ((rc = vo_write_calib(ctx, p * n + q, 1, &ctx->seq_cal_next[p * n + q])) ||
                (rc = vo_write_params(ctx, p * n + q, 1, &ctx->seq_par_next[p * n + q])))
                return rc;
            ctx->seq_cal_due[p * n + q] = 0;
        }
    for (int i = 0; i < n_start; i++) {
        const int q = starts[i].slot;
        const CamCalib c = vo_calib_from(starts[i].P_l, starts[i].P_r);
        const UnitParams e = vo_unit_params(ctx->seq_par[q]);
        if ((rc = vo_write_calib(ctx, p * n + q, 1, &c)) || (rc = vo_write_params(ctx, p * n + q, 1, &e))) return rc;
        ctx->seq_cal_next[(1 - p) * n + q] = c;
        ctx->seq_par_next[(1 - p) * n + q] = e;
        ctx->seq_cal_due[(1 - p) * n + q] = 1;
        VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_feat_cnt + 2 * q, 0, 2 * sizeof(int), ctx->stream));
    }
    // the live words of parity p: a sequence retired by this or an earlier submission (or started by this one) stops
    // working from this frame on, a started one works from the next; the other parity's word is still read by the frame
    // in flight, and is written by the next submission
    for (int q = 0; q < n; q++) {
        const char want = st && st[q] ? SEQ_STARTED : ctx->seq_retired[q] ? 0 : 1;
        if ((ctx->seq_live[p * n + q] == 1) != (want == 1))
            VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_seq_live + p * n + q, want == 1 ? 1 : 0, sizeof(int), ctx->stream));
        ctx->seq_live[p * n + q] = want;
    }
    // geometry entries of the image slot s1 for the pairs of started sequences staged into it, on stream gs.  Host pairs:
    // on the front stream here (their upload reads no entry; the front stage's kernels do).  Device pairs: the conversion
    // on the copy stream reads them, and it is not ordered after this point of the front stream (it follows fork_ev,
    // recorded before the wait for seq_back_ev[p] above, so that it does not queue behind frame k-2's pose solve); they are
    // written on the copy stream after its waits below instead.  Either way every earlier reader of slot s1's entries (the
    // front stage of frame k-2, which seq_front_ev[p] covers) is done, and every later one (the conversion, the front
    // stage of this frame) follows the write.
    auto write_geo = [&](cudaStream_t gs) {
        for (int q = 0; ctx->seq_sized && q < n; q++)
            if (ctx->seq_geo_due[q] && in.left(q)) {
                const PlaneGeom g = vo_plane_geom(ctx, ctx->seq_w[q], ctx->seq_h[q]), gg[2] = {g, g};
                const int rw = vo_write_geo(ctx, 2 * n * s1 + 2 * q, 2, gg, gs);
                if (rw) return rw;
                ctx->seq_geo_due[q]--;
            }
        return VO_OK;
    };
    if (!in.device && (rc = write_geo(ctx->stream))) return rc;
    if (bgr) {
        // colour frames share one staging buffer: upload + convert stay on the front stream
        if ((rc = stage_pairs(ctx, s1, in, ctx->stream))) return rc;
    } else {
        // image slot s1 (of three) was last read, as the previous pair, by the front stage of the frame before the one
        // now running: that frame has this frame's buffer parity, and its seq_front_ev[p] record is still the
        // current one (it is re-recorded below).  So this copy (or the conversion of a device pair, launched outside the
        // frame graph because its source pointers change every frame) runs under the front stage of the frame in flight.
        // (No ordering against the caller's stream is needed for host pairs: vo_seq_begin synchronises, and every later
        // access to the image slots is made by this file and ordered through these events.  A host upload must not wait
        // for fork_ev: that would queue its H2D behind the previous front stage.)
        cudaStream_t sc = ctx->lane[1].side;
        VO_CUDA_CHECK(cudaStreamWaitEvent(sc, ctx->seq_front_ev[p], 0));
        if (in.device) VO_CUDA_CHECK(cudaStreamWaitEvent(sc, ctx->fork_ev, 0));
        if (in.device && (rc = write_geo(sc))) return rc;
        if ((rc = stage_pairs(ctx, s1, in, sc))) return rc;
        // The join is also the release of device images: the caller's later work on ctx->stream is ordered after the
        // conversion, the last read of the images.
        VO_CUDA_CHECK(cudaEventRecord(ctx->lane[1].join, sc));
        VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->lane[1].join, 0));
    }
    GraphKey key{};
    key.kind = GraphKey::SEQ_FRONT; key.s = ctx->stream; key.tma = ctx->lk_use_tma;
    key.slot = s0; key.parity = p; key.bgr = bgr;
    // the LK launch bound: the largest bucket grid of the sequences' sizes, which a new set of sizes inside the same
    // envelope, or a start, can raise (the sizes themselves are in the geometry table, not in the graph)
    key.max_pts = ctx->seq_lk_bound;
    if ((rc = vo_run_graph(ctx, key, [&] { return seq_front(ctx, s0, s1, p, bgr); }))) return rc;
    VO_CUDA_CHECK(cudaEventRecord(ctx->seq_front_ev[p], ctx->stream));
    // back stage: after this frame's front stage; after the previous frame's back stage by stream order
    cudaStream_t sb = ctx->lane[0].side;
    VO_CUDA_CHECK(cudaStreamWaitEvent(sb, ctx->seq_front_ev[p], 0));
    key = GraphKey{};
    key.kind = GraphKey::SEQ_BACK; key.s = sb; key.tma = ctx->lk_use_tma; key.parity = p;
    if ((rc = vo_run_graph(ctx, key, [&] { return seq_back(ctx, p); }))) return rc;
    // a started sequence's next frame solves from zeros: after k_seq_finish of this frame copied the slot's translation
    for (int i = 0; i < n_start; i++)
        VO_CUDA_CHECK(cudaMemsetAsync(ctx->d_tprev + 3 * (size_t)((1 - p) * n + starts[i].slot), 0, 3 * sizeof(double), sb));
    const int u0 = p * n;
    const SeqPinned pin = seq_pinned(ctx, n);
    // (vo_mseq_wait_device reads the records, error words and essential results on the device: no copies)
    if (!ctx->seq_dres) {
        VO_CUDA_CHECK(cudaMemcpyAsync(pin.rec + u0, ctx->d_results + u0, n * sizeof(vo_unit_result_dev), cudaMemcpyDeviceToHost, sb));
        VO_CUDA_CHECK(cudaMemcpyAsync(pin.err + u0, ctx->d_seq_err + 1 + u0, n * sizeof(int), cudaMemcpyDeviceToHost, sb));
        if (ctx->seq_mono) {            // the n results, one per scratch block, into n consecutive records: one strided copy
            EssArgs e;
            seq_ess_args(ctx, u0, n, e);
            VO_CUDA_CHECK(cudaMemcpy2DAsync(pin.ess + u0, sizeof(EssResult), e.result, e.result_stride, sizeof(EssResult), n,
                                            cudaMemcpyDeviceToHost, sb));
        }
    }
    VO_CUDA_CHECK(cudaEventRecord(ctx->seq_back_ev[p], sb));
    ctx->seq_slot = s1;                 // imageLeft_t0 = imageLeft_t1 (main.cpp:157-158)
    ctx->seq_submitted++;
    ctx->seq_inflight++;
    return VO_OK;
}

// Waits for the oldest submission (who / multi: the calling entry point; want_mono: vo_[m]seq_wait_mono); per sequence q:
// out[q], status[q] (multi only: VO_OK, VO_E_CAPACITY for glue error bits, VO_MSEQ_RETIRED), frame_pose integrated, with
// pts4 the four point lists at pts4 + 4 * pts_cap * q, and with want_mono mono[q] and the essential mask at
// ess_mask + mask_cap * q.  Returns the first status that is an error (the single-sequence mode reports its frame this
// way), else VO_OK.
static int seq_wait(vo_ctx* ctx, const char* who, bool multi, bool want_mono, vo_unit_result* out, int* status, vo_mono_result* mono,
                    uint8_t* ess_mask, int mask_cap, vo_point2f* pts4, int pts_cap)
{
    if (!ctx) return VO_E_INVALID;
    int rc;
    if ((rc = seq_frame_check(ctx, who, multi, SEQ_WAIT))) return rc;
    if (ctx->seq_dres) {
        vo_set_error(ctx, "%s: the sequences were begun with VO_MSEQ_DEVICE_RESULTS: use vo_mseq_wait_device", who);
        return VO_E_INVALID;
    }
    if (!out || (multi && !status) || (want_mono && !mono)) { vo_set_error(ctx, "%s: null result", who); return VO_E_INVALID; }
    if (want_mono && !ctx->seq_mono) {
        vo_set_error(ctx, multi ? "%s: the sequences were begun without the flag VO_MSEQ_MONO_ROTATION"
                                : "%s: the sequence was begun without the option \"mono_rotation\"", who);
        return VO_E_INVALID;
    }
    int single_status;
    if (!multi) status = &single_status;
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const int p = (int)((ctx->seq_submitted - ctx->seq_inflight) & 1);      // the parity of the oldest frame in flight
    VO_CUDA_CHECK(cudaEventSynchronize(ctx->seq_back_ev[p]));
    const int n = ctx->seq_n, u0 = p * n;
    const SeqPinned pin = seq_pinned(ctx, n);
    ctx->seq_inflight--;
    const size_t cs = (size_t)ctx->units * ctx->cap;
    cudaStream_t sb = ctx->lane[0].side;
    bool copies = false;
    for (int q = 0; q < n; q++) {
        if (ctx->seq_live[u0 + q] != 1) {               // retired (or never started), or started by this submission: nothing ran
            memset(&out[q], 0, sizeof(out[q]));
            if (mono) memset(&mono[q], 0, sizeof(mono[q]));
            status[q] = VO_MSEQ_RETIRED;
            if (ctx->seq_live[u0 + q] == SEQ_STARTED) {     // the new sequence's frame_pose starts here (main.cpp:90)
                status[q] = VO_MSEQ_STARTED;
                double* pose = ctx->seq_pose.data() + 16 * q;
                for (int i = 0; i < 16; i++) pose[i] = i % 5 == 0 ? 1.0 : 0.0;
            }
            continue;
        }
        const vo_unit_result_dev r = pin.rec[u0 + q];
        const int err = pin.err[u0 + q];
        memcpy(&out[q], &r, sizeof(r));
        // main.cpp:196-208.  The reference ignores solvePnPRansac's return value: when RANSAC finds no model, rvec stays 0
        // (R = I) and `translation` keeps the carried value, and the main loop still integrates that motion.  With
        // mono_rotation, where cv::findEssentialMat / cv::recoverPose would throw (n < 5, no E with more than 4 inliers,
        // n == 5 with other than one candidate) the frame is reported (R = I) and not integrated, like an n < 4 PnP frame.
        const EssResult& ess = pin.ess[u0 + q];
        const bool mono_ok = !ctx->seq_mono || ess.status == ESS_OK;
        if ((r.pnp_status == VO_OK || r.pnp_status == VO_PNP_NO_MODEL) && mono_ok) vo_pose_step(ctx->seq_pose.data() + 16 * q, r.R, r.tvec);
        if (mono) {
            vo_mono_result& m = mono[q];
            m.status = mono_ok ? VO_OK : VO_E_TOO_FEW_POINTS;
            m.n_inliers = ess.n_inliers; m.ransac_iters = ess.iters; m.n_good = ess.n_good;
            for (int k = 0; k < 9; k++) m.R[k] = ess.R[k];
            for (int k = 0; k < 3; k++) m.t[k] = ess.t[k];
        }
        // the frame's point lists (and essential mask) stay in its buffer units until the frame after next is submitted
        const size_t uo = (size_t)(u0 + q) * ctx->cap;
        if (pts4 && pts_cap > 0 && r.n_valid > 0) {
            const int m = r.n_valid < pts_cap ? r.n_valid : pts_cap;
            for (int k = 0; k < 4; k++)
                VO_CUDA_CHECK(cudaMemcpyAsync(pts4 + (size_t)(4 * q + k) * pts_cap, ctx->d_valid4 + k * cs + uo, (size_t)m * sizeof(float2),
                                              cudaMemcpyDeviceToHost, sb));
            copies = true;
        }
        if (ess_mask && mask_cap > 0 && r.n_valid > 0) {
            EssArgs e;
            seq_ess_args(ctx, u0 + q, 1, e);
            const int m = r.n_valid < mask_cap ? r.n_valid : mask_cap;
            VO_CUDA_CHECK(cudaMemcpyAsync(ess_mask + (size_t)mask_cap * q, e.mask, (size_t)m, cudaMemcpyDeviceToHost, sb));
            copies = true;
        }
        // bit 8 (a tracked point outside the bucket grid: undefined behaviour in the reference, dropped here) is not an error
        status[q] = VO_OK;
        if (err & ~8) {
            status[q] = VO_E_CAPACITY;
            if (rc == VO_OK) {
                if (ctx->seq_multi) vo_set_error(ctx, "vo_mseq: glue kernel error bits 0x%x of sequence %d (1/2: capacity, 4: bucket grid)", err, q);
                else vo_set_error(ctx, "vo_seq: glue kernel error bits 0x%x of this frame (1/2: capacity, 4: bucket grid)", err);
                rc = VO_E_CAPACITY;
            }
        }
    }
    if (copies) VO_CUDA_CHECK(cudaStreamSynchronize(sb));
    return rc;
}

static_assert(sizeof(vo_unit_result) == sizeof(vo_unit_result_dev), "k_seq_collect writes vo_unit_result records");

// VO_E_INVALID + message unless p is NULL or device (managed) memory of the context's GPU
static int seq_check_dptr(vo_ctx* ctx, const char* who, const char* name, const void* p)
{
    if (!p) return VO_OK;
    cudaPointerAttributes a;
    const cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) { cudaGetLastError(); vo_set_error(ctx, "%s: %s: not a CUDA pointer (%s)", who, name, cudaGetErrorString(e)); return VO_E_INVALID; }
    if (a.type == cudaMemoryTypeManaged) return VO_OK;
    if (a.type != cudaMemoryTypeDevice || a.device != ctx->device) {
        vo_set_error(ctx, "%s: %s is not device memory of GPU %d", who, name, ctx->device);
        return VO_E_INVALID;
    }
    return VO_OK;
}

// vo_mseq_wait_device: the oldest submission retired by ONE k_seq_collect launch on the context's stream, after the
// caller's work there and after that submission's back stage (seq_back_ev of its parity; the next submission's back stage
// on the side stream is not waited for).  The stream order also covers the unit buffers: the next submission of the same
// parity, which overwrites them, queues its front stage on the context's stream after this launch, and its back stage
// after that front stage.  The host only moves its bookkeeping on.
static int seq_wait_device(vo_ctx* ctx, const char* who, const vo_mseq_dresults* r)
{
    if (!ctx) return VO_E_INVALID;
    int rc;
    if ((rc = seq_frame_check(ctx, who, true, SEQ_WAIT))) return rc;
    if (!ctx->seq_dres) {
        vo_set_error(ctx, "%s: the sequences were begun without the flag VO_MSEQ_DEVICE_RESULTS (use vo_mseq_wait)", who);
        return VO_E_INVALID;
    }
    if (!r) { vo_set_error(ctx, "%s: null result table", who); return VO_E_INVALID; }
    const bool lists = r->pts4 || r->points3d || r->inliers || r->ess_mask;
    if (r->pts_cap < 0 || (lists && r->pts_cap == 0)) {
        vo_set_error(ctx, "%s: pts_cap = %d with point arrays", who, r->pts_cap);
        return VO_E_INVALID;
    }
    if ((r->mono || r->ess_mask) && !ctx->seq_mono) {
        vo_set_error(ctx, "%s: mono / ess_mask: the sequences were begun without the flag VO_MSEQ_MONO_ROTATION", who);
        return VO_E_INVALID;
    }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const struct { const char* name; const void* p; } ptrs[] = {
        {"status", r->status}, {"records", r->records}, {"frame_pose", r->frame_pose}, {"pts4", r->pts4},
        {"points3d", r->points3d}, {"inliers", r->inliers}, {"mono", r->mono}, {"ess_mask", r->ess_mask}};
    for (const auto& x : ptrs)
        if ((rc = seq_check_dptr(ctx, who, x.name, x.p))) return rc;
    const int n = ctx->seq_n;
    const int p = (int)((ctx->seq_submitted - ctx->seq_inflight) & 1);      // the parity of the oldest frame in flight
    const int u0 = p * n;
    const size_t cs = (size_t)ctx->units * ctx->cap, uo = (size_t)u0 * ctx->cap;
    CollectArgs a;
    memset(&a, 0, sizeof(a));
    a.res = ctx->d_results + u0; a.err = ctx->d_seq_err + 1 + u0; a.cap = ctx->cap;
    a.valid4 = ctx->d_valid4 + uo; a.plane_stride = cs;
    a.X = ctx->d_X + uo; a.inliers = ctx->d_inliers + uo;
    if (ctx->seq_mono) {
        EssArgs e;
        seq_ess_args(ctx, u0, n, e);
        a.ess = e.result; a.ess_mask = e.mask; a.ess_stride = ctx->seq_ess_bytes;
    }
    a.pose = ctx->d_seq_pose;
    a.status = r->status; a.records = (vo_unit_result_dev*)r->records; a.pose_out = r->frame_pose; a.pts_cap = r->pts_cap;
    a.pts4 = (float2*)r->pts4; a.points3d = (float3*)r->points3d; a.inliers_out = r->inliers; a.mono = r->mono;
    a.mask_out = r->ess_mask;
    for (int q = 0; q < n; q++) a.mode[q] = (unsigned char)ctx->seq_live[u0 + q];
    VO_CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->seq_back_ev[p], 0));
    ctx->launches += vo_launch_seq_collect(a, n, ctx->stream);
    VO_CUDA_CHECK(cudaGetLastError());
    ctx->seq_inflight--;
    return VO_OK;
}

// currentVOFeatures and the carried translation of sequence q (after the frames in flight)
static int seq_state(vo_ctx* ctx, const char* who, bool multi, int q, vo_point2f* points, int32_t* ages, int cap, int* n_points,
                     int* n_ages, double t_out[3])
{
    if (!ctx) return VO_E_INVALID;
    int rc;
    if ((rc = seq_frame_check(ctx, who, multi, SEQ_QUERY))) return rc;
    if (q < 0 || q >= ctx->seq_n) { vo_set_error(ctx, "%s: bad sequence index %d", who, q); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    if ((rc = seq_drain(ctx))) return rc;
    int cnt[2] = {0, 0};
    VO_CUDA_CHECK(cudaMemcpyAsync(cnt, ctx->d_feat_cnt + 2 * q, 2 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    // the translation the NEXT frame will start from lives in the next frame's buffer parity
    const size_t next = (size_t)(ctx->seq_submitted & 1) * ctx->seq_n + q;
    if (t_out) VO_CUDA_CHECK(cudaMemcpyAsync(t_out, ctx->d_tprev + 3 * next, 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (n_points) *n_points = cnt[0];
    if (n_ages) *n_ages = cnt[1];
    const size_t fo = (size_t)q * ctx->feat_cap;
    if (points && cnt[0] > 0) VO_CUDA_CHECK(cudaMemcpyAsync(points, ctx->d_feat_pts + fo, (size_t)(cnt[0] < cap ? cnt[0] : cap) * sizeof(float2), cudaMemcpyDeviceToHost, ctx->stream));
    if (ages && cnt[1] > 0) VO_CUDA_CHECK(cudaMemcpyAsync(ages, ctx->d_feat_ages + fo, (size_t)(cnt[1] < cap ? cnt[1] : cap) * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}

// ---- one sequence (vo_seq_*) ---------------------------------------------------------------------------------------
extern "C" int vo_seq_begin(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const uint8_t* left0,
                            const uint8_t* right0, size_t pitch)
{
    return vo_seq_begin_ex(ctx, w, h, P_l, P_r, left0, right0, pitch, 1);
}

extern "C" int vo_seq_begin_ex(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const uint8_t* left0,
                               const uint8_t* right0, size_t pitch, int channels)
{
    const SeqPairs in = host_pairs(&left0, &right0, &pitch, channels);
    return seq_begin(ctx, "vo_seq_begin", false, 1, 0, &w, &h, P_l, P_r, &in);
}

extern "C" int vo_seq_begin_device(vo_ctx* ctx, int w, int h, const float P_l[12], const float P_r[12], const vo_dimage* left0,
                                   const vo_dimage* right0)
{
    const SeqPairs in = device_pairs(left0, right0);
    return seq_begin(ctx, "vo_seq_begin_device", false, 1, 0, &w, &h, P_l, P_r, &in);
}

extern "C" int vo_seq_submit(vo_ctx* ctx, const uint8_t* left1, const uint8_t* right1, size_t pitch, int channels)
{
    return seq_submit(ctx, "vo_seq_submit", false, host_pairs(&left1, &right1, &pitch, channels));
}

extern "C" int vo_seq_submit_device(vo_ctx* ctx, const vo_dimage* left1, const vo_dimage* right1)
{
    return seq_submit(ctx, "vo_seq_submit_device", false, device_pairs(left1, right1));
}

extern "C" int vo_seq_wait(vo_ctx* ctx, vo_unit_result* out, vo_point2f* pts4, int pts_cap)
{
    return seq_wait(ctx, "vo_seq_wait", false, false, out, nullptr, nullptr, nullptr, 0, pts4, pts_cap);
}

extern "C" int vo_seq_wait_mono(vo_ctx* ctx, vo_unit_result* out, vo_mono_result* mono, uint8_t* ess_mask, int mask_cap,
                                vo_point2f* pts4, int pts_cap)
{
    return seq_wait(ctx, "vo_seq_wait_mono", false, true, out, nullptr, mono, ess_mask, mask_cap, pts4, pts_cap);
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
    return seq_state(ctx, "vo_seq_state", false, 0, points, ages, cap, n_points, n_ages, t_out);
}

// ---- several sequences in lockstep (vo_mseq_*) ---------------------------------------------------------------------
extern "C" int vo_mseq_begin(vo_ctx* ctx, int n_seq, int w, int h, const float P_l[12], const float P_r[12], const uint8_t* const* left0,
                             const uint8_t* const* right0, size_t pitch, int channels)
{
    return vo_mseq_begin_ex(ctx, n_seq, w, h, P_l, P_r, left0, right0, pitch, channels, 0);
}

// one calibration for every sequence: vo_mseq_begin_calib with the matrices repeated
extern "C" int vo_mseq_begin_ex(vo_ctx* ctx, int n_seq, int w, int h, const float P_l[12], const float P_r[12],
                                const uint8_t* const* left0, const uint8_t* const* right0, size_t pitch, int channels, int flags)
{
    if (!ctx) return VO_E_INVALID;
    if (!P_l || !P_r || n_seq < 1 || n_seq > VO_MSEQ_MAX)        // refused below with its message
        return vo_mseq_begin_calib(ctx, n_seq, w, h, P_l, P_r, left0, right0, pitch, channels, flags);
    std::vector<float> Pl(12 * (size_t)n_seq), Pr(12 * (size_t)n_seq);
    for (int q = 0; q < n_seq; q++) {
        memcpy(Pl.data() + 12 * q, P_l, 12 * sizeof(float));
        memcpy(Pr.data() + 12 * q, P_r, 12 * sizeof(float));
    }
    return vo_mseq_begin_calib(ctx, n_seq, w, h, Pl.data(), Pr.data(), left0, right0, pitch, channels, flags);
}

// one image size and row pitch for every sequence: vo_mseq_begin_sized with them repeated
extern "C" int vo_mseq_begin_calib(vo_ctx* ctx, int n_seq, int w, int h, const float* P_l, const float* P_r,
                                   const uint8_t* const* left0, const uint8_t* const* right0, size_t pitch, int channels, int flags)
{
    const int n = n_seq >= 1 && n_seq <= VO_MSEQ_MAX ? n_seq : 1;     // other counts are refused with their message
    const std::vector<int> ws(n, w), hs(n, h);
    const std::vector<size_t> ps(n, pitch);
    const SeqPairs in = host_pairs(left0, right0, ps.data(), channels);
    return seq_begin(ctx, "vo_mseq_begin", true, n_seq, flags, ws.data(), hs.data(), P_l, P_r, &in);
}

extern "C" int vo_mseq_begin_sized(vo_ctx* ctx, int n_seq, const int* w, const int* h, const float* P_l, const float* P_r,
                                   const uint8_t* const* left0, const uint8_t* const* right0, const size_t* pitch, int channels,
                                   int flags)
{
    const SeqPairs in = host_pairs(left0, right0, pitch, channels);
    return seq_begin(ctx, "vo_mseq_begin_sized", true, n_seq, flags, w, h, P_l, P_r, &in);
}

// Host state only: a slot's setting reaches the device when a begin or start of the slot writes its units' entries
extern "C" int vo_mseq_params(vo_ctx* ctx, int first_slot, int n, const vo_params* p)
{
    if (!ctx) return VO_E_INVALID;
    if (first_slot < 0 || n <= 0 || first_slot > VO_MSEQ_MAX - n) {
        vo_set_error(ctx, "vo_mseq_params: slots [%d, %d) outside [0, %d)", first_slot, first_slot + n, VO_MSEQ_MAX);
        return VO_E_INVALID;
    }
    for (int i = 0; p && i < n; i++) {
        char what[32];
        snprintf(what, sizeof(what), "slot %d", first_slot + i);
        const int rc = vo_check_unit_params(ctx, "vo_mseq_params", what, p[i]);
        if (rc) return rc;
    }
    for (int i = 0; i < n; i++) ctx->slot_par[first_slot + i] = p ? p[i] : ctx->p;
    return VO_OK;
}

// one row pitch for every image: vo_mseq_submit_sized with it repeated (it must cover every live sequence's width)
extern "C" int vo_mseq_submit(vo_ctx* ctx, const uint8_t* const* left1, const uint8_t* const* right1, size_t pitch, int channels)
{
    const std::vector<size_t> ps(ctx && ctx->seq_active && ctx->seq_multi ? ctx->seq_n : 1, pitch);
    return seq_submit(ctx, "vo_mseq_submit", true, host_pairs(left1, right1, ps.data(), channels));
}

extern "C" int vo_mseq_submit_sized(vo_ctx* ctx, const uint8_t* const* left1, const uint8_t* const* right1, const size_t* pitch,
                                    int channels)
{
    return seq_submit(ctx, "vo_mseq_submit_sized", true, host_pairs(left1, right1, pitch, channels));
}

// n_slots empty slots at the envelope max_w x max_h; sequences come in through vo_mseq_submit_start
extern "C" int vo_mseq_open(vo_ctx* ctx, int n_slots, int max_w, int max_h, int flags)
{
    const int n = n_slots >= 1 && n_slots <= VO_MSEQ_MAX ? n_slots : 1;     // other counts are refused with their message
    const std::vector<int> ws(n, max_w), hs(n, max_h);
    return seq_begin(ctx, "vo_mseq_open", true, n_slots, flags, ws.data(), hs.data(), nullptr, nullptr, nullptr);
}

extern "C" int vo_mseq_submit_start(vo_ctx* ctx, const uint8_t* const* left1, const uint8_t* const* right1, const size_t* pitch,
                                    int channels, int n_start, const vo_mseq_start* starts)
{
    return seq_submit(ctx, "vo_mseq_submit_start", true, host_pairs(left1, right1, pitch, channels), n_start, starts);
}

extern "C" int vo_mseq_begin_device(vo_ctx* ctx, int n_seq, const int* w, const int* h, const float* P_l, const float* P_r,
                                    const vo_dimage* left0, const vo_dimage* right0, int flags)
{
    const SeqPairs in = device_pairs(left0, right0);
    return seq_begin(ctx, "vo_mseq_begin_device", true, n_seq, flags, w, h, P_l, P_r, &in);
}

extern "C" int vo_mseq_submit_device(vo_ctx* ctx, const vo_dimage* left1, const vo_dimage* right1, int n_start,
                                     const vo_mseq_start* starts)
{
    return seq_submit(ctx, "vo_mseq_submit_device", true, device_pairs(left1, right1), n_start, starts);
}

extern "C" int vo_mseq_wait(vo_ctx* ctx, vo_unit_result* out, int* status, vo_point2f* pts4, int pts_cap)
{
    return seq_wait(ctx, "vo_mseq_wait", true, false, out, status, nullptr, nullptr, 0, pts4, pts_cap);
}

extern "C" int vo_mseq_wait_mono(vo_ctx* ctx, vo_unit_result* out, int* status, vo_mono_result* mono, uint8_t* ess_mask, int mask_cap,
                                 vo_point2f* pts4, int pts_cap)
{
    return seq_wait(ctx, "vo_mseq_wait_mono", true, true, out, status, mono, ess_mask, mask_cap, pts4, pts_cap);
}

extern "C" int vo_mseq_wait_device(vo_ctx* ctx, const vo_mseq_dresults* r)
{
    return seq_wait_device(ctx, "vo_mseq_wait_device", r);
}

extern "C" int vo_mseq_pose(vo_ctx* ctx, int q, double frame_pose[16])
{
    if (!ctx) return VO_E_INVALID;
    int rc;
    if ((rc = seq_frame_check(ctx, "vo_mseq_pose", true, SEQ_QUERY))) return rc;
    if (q < 0 || q >= ctx->seq_n || !frame_pose) { vo_set_error(ctx, "vo_mseq_pose: bad argument"); return VO_E_INVALID; }
    if (ctx->seq_dres) {            // after the last vo_mseq_wait_device's k_seq_collect (the context's stream)
        VO_CUDA_CHECK(cudaSetDevice(ctx->device));
        if ((rc = seq_drain(ctx))) return rc;
        VO_CUDA_CHECK(cudaMemcpyAsync(frame_pose, ctx->d_seq_pose + 16 * (size_t)q, 16 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        return VO_OK;
    }
    memcpy(frame_pose, ctx->seq_pose.data() + 16 * (size_t)q, 16 * sizeof(double));
    return VO_OK;
}

extern "C" int vo_mseq_state(vo_ctx* ctx, int q, vo_point2f* points, int32_t* ages, int cap, int* n_points, int* n_ages, double t_out[3])
{
    return seq_state(ctx, "vo_mseq_state", true, q, points, ages, cap, n_points, n_ages, t_out);
}
