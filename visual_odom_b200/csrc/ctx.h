// ctx.h -- the library context (device-resident state shared by every entry point)
#pragma once
#include "common.cuh"
#include "lk_ring.h"
#include "filter.h"
#include "fast.h"
#include "pnp.h"
#include "seq.h"
#include "ess.h"
#include "../../include/vo_b200.h"
#include <vector>
#include <functional>
#include <stdarg.h>
#define LK_QUEUES 32
#define VO_DIST_BUCKET 4       // posted steps per collective
#define VO_DIST_NB 4           // buckets (ring)
#define VO_LANES 3            // submissions in flight, each with its own side stream / partition streams / events

// what a cached CUDA graph was captured for: its kind, the stream (the LK work queue is that stream's), the LK staging,
// and the kind's own fields (the others stay zero)
struct GraphKey {
    enum Kind { BATCH_RANGE, SEQ_FRONT, SEQ_BACK } kind;
    cudaStream_t s;
    bool tma;
    int u0, n, max_pts; bool detect;        // BATCH_RANGE: the unit range, its feature bound, on-GPU detection
                                            // (SEQ_FRONT: max_pts = the LK launch bound, the sequences' largest bucket grid)
    int slot, parity; bool bgr;             // SEQ_FRONT / SEQ_BACK: image slot of the previous pairs, buffer parity, colour input
};

struct vo_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    vo_params p;
    char err[1024] = {0};
    long long launches = 0;
    int sm_count = 0;

    // ---- geometry of the currently allocated batch state -----------------------------------
    int w = 0, h = 0;             // image size
    int units = 0;                // allocated work-unit slots
    int cap = 0;                  // feature capacity per unit
    PyrGeom pg;                   // device plane pointers per level
    LkMaps maps;                  // TMA descriptors per level
    // calibration table (part of the batch state, so its address is fixed for as long as any captured graph lives):
    // entry 0 is the stage calls' (vo_triangulate, vo_pnp_ransac), entry 1 + u buffer unit u's.  The kernels read their
    // unit's entry, so captured graphs carry no calibration and a table write needs no graph drop.  cal mirrors it.
    CamCalib* d_cal_tab = nullptr;      // [1 + units]
    CamCalib* d_cal = nullptr;          // d_cal_tab + 1: indexed by buffer unit
    std::vector<CamCalib> cal;          // [1 + units] host copy (kept across re-allocations of the batch state)
    // parameter table (the same layout and life as the calibration table): entry 0 the stage calls' (always the context's
    // vo_params), entry 1 + u buffer unit u's tracking parameters (vo_mseq_params, vo_batch_params).  par mirrors it.
    UnitParams* d_par_tab = nullptr;    // [1 + units]
    UnitParams* d_par = nullptr;        // d_par_tab + 1: indexed by buffer unit
    std::vector<UnitParams> par;        // [1 + units] host copy (kept across re-allocations of the batch state)
    // vo_mseq_params: each slot's setting, which the begin and start calls of the slot read ([VO_MSEQ_MAX], the context's
    // vo_params until set)
    std::vector<vo_params> slot_par;
    // geometry table (the same life as d_cal_tab): one entry per raw image plane, its own size per level and raw pitch.
    // w / h above are then the envelope of the sizes; only runs of several sizes (vo_mseq_begin_sized) point kernels at
    // it, every other path uses the launch-wide sizes.  Entries start out as w x h.  geo mirrors it.
    PlaneGeom* d_geo = nullptr;         // [units * 4]
    std::vector<PlaneGeom> geo;

    // ---- device buffers ---------------------------------------------------------------------
    uint8_t* d_raw = nullptr;           // [units*4][h*w] raw images (a smaller image: its own rows packed from the plane start)
    const uint8_t** d_raw_tab = nullptr;// [units*4] pointers into d_raw
    vo_dimage* d_ingest_tab = nullptr;  // [units*4] descriptors of caller device images, per raw plane (staged per submission)
    float2* d_pts_in = nullptr;         // [units][cap]
    int* d_npts = nullptr;              // [units]
    float2* d_pts_out = nullptr;        // [4][units][cap]
    uint8_t* d_status = nullptr;        // [4][units][cap]
    float* d_err = nullptr;             // [4][units][cap]
    int* d_ages_in = nullptr;           // [units][cap]
    int* d_ages_out = nullptr;          // [units][cap]
    float2* d_kept5 = nullptr;          // [5][units][cap]
    int* d_idx3 = nullptr;              // [units][cap]
    int* d_n3 = nullptr;                // [units]
    float2* d_valid4 = nullptr;         // [4][units][cap]
    int* d_idx5 = nullptr;              // [units][cap]
    int* d_n5 = nullptr;                // [units]
    // FAST
    uint8_t* d_score = nullptr;         // [units][h*w]
    uint16_t* d_rowbuf = nullptr;       // [units][h][w]
    int* d_rowcount = nullptr;          // [units][h]
    int* d_rowoff = nullptr;            // [units][h]
    int* d_ndet = nullptr;              // [units]
    float2* d_corners = nullptr;        // [units][corner_cap]
    float* d_resp = nullptr;            // [units][corner_cap]
    int* d_want = nullptr;              // [units] features to select (batched path)
    int corner_cap = 0;
    // triangulation + PnP
    float3* d_X = nullptr;              // [units][cap]
    double* d_tprev = nullptr;          // [units][3]
    PnpState* d_pnp_state = nullptr;    // [units]
    int* d_subsets = nullptr;           // [units][iters][5]
    double* d_models = nullptr;         // [units][iters][12]
    int* d_counts = nullptr;            // [units][iters]
    int* d_inliers = nullptr;           // [units][cap]
    vo_unit_result_dev* d_results = nullptr;   // [units]
    // sequence mode (seq.cu): the reference main loop's state, device resident, for seq_n sequences run in lockstep
    // (vo_seq_*: one; vo_mseq_*: n_seq).  Sequence q at buffer parity p uses work unit p * seq_n + q.
    float2* d_feat_pts = nullptr;       // [seq_n_cap][feat_cap] currentVOFeatures.points
    int* d_feat_ages = nullptr;         // [seq_n_cap][feat_cap] currentVOFeatures.ages (may be longer than points)
    int* d_feat_cnt = nullptr;          // [seq_n_cap][2] sizes of the two vectors
    int* d_bucket = nullptr;            // [seq_n_cap][bucket_cap] scratch of bucketingFeatures (k_seq_bucket)
    int* d_seq_err = nullptr;           // [1 + 2 * seq_n_cap] error bits of the glue kernels, [1 + unit] per frame
    int* d_seq_live = nullptr;          // [2 * seq_n_cap] per unit: 0 once its sequence is retired (vo_mseq_submit)
    void* d_seq_state = nullptr;        // the one allocation behind the six arrays above (freed with the batch state)
    int seq_n_cap = 0;                  // sequences those arrays hold
    int feat_cap = 0;
    // ints of bucketing scratch per sequence: a grid of nb cells takes nb * (k + 1) at features_per_bucket k, and every
    // run the begin and start calls accept has nb * k <= max_features, so nb <= max_features and nb * (k + 1) <=
    // 2 * max_features whatever each sequence's k (vo_create)
    size_t bucket_cap = 0;
    bool seq_active = false;
    bool seq_multi = false;             // begun with vo_mseq_begin (the vo_seq_* frame calls are refused, and vice versa)
    int seq_n = 1;                      // sequences of the running sequence mode
    bool seq_sized = false;             // the sequences' image sizes differ (planes are envelope-sized, kernels read d_geo)
    std::vector<int> seq_w, seq_h;      // [seq_n] each sequence's image size
    std::vector<vo_params> seq_par;     // [seq_n] each sequence's parameters (its slot's setting when it began or started)
    int seq_slot = 0;                   // image slot holding the previous stereo pairs: raw/pyramid planes
                                        // 2 * seq_n * slot + 2q (left), + 1 (right) of sequence q
    int seq_inflight = 0;               // frames submitted and not yet waited for (<= 2)
    long long seq_submitted = 0;        // frames submitted since vo_seq_begin (frame k uses buffer parity k & 1)
    cudaEvent_t seq_front_ev[2] = {nullptr, nullptr}, seq_back_ev[2] = {nullptr, nullptr};
    std::vector<double> seq_pose;       // [seq_n][16] frame_pose of main.cpp:90, integrated per push
    std::vector<char> seq_retired;      // [seq_n] no sequence runs in the slot: retired by a NULL pair (vo_mseq_submit), or
                                        // never started (vo_mseq_open)
    std::vector<char> seq_live;         // [2 * seq_n] d_seq_live as the frame in flight in each parity saw it: 0 not running,
                                        // 1 running, SEQ_STARTED (host only, the device word is 0) its sequence started there
    // results into device memory (flag VO_MSEQ_DEVICE_RESULTS, vo_mseq_wait_device): frame_pose lives in d_seq_pose
    // ([VO_MSEQ_MAX][16], allocated at the first such begin) and k_seq_collect integrates it.  The host no longer waits for
    // a submission, so the descriptor table entries of image slot s (pinned) are rewritten only after seq_tab_ev[s], recorded
    // after their copy to the device.
    bool seq_dres = false;
    double* d_seq_pose = nullptr;
    cudaEvent_t seq_tab_ev[3] = {nullptr, nullptr, nullptr};
    int seq_lk_bound = 0;               // the LK launch bound: the largest bucket grid of the run's sizes (raised by starts)
    std::vector<CamCalib> seq_cal_next; // [2 * seq_n] calibration and parameter entries of started sequences that the
    std::vector<UnitParams> seq_par_next;   // frame in flight still reads: written by the next submission of that buffer
    std::vector<char> seq_cal_due;      // parity
    std::vector<char> seq_geo_due;      // [seq_n] image slots whose geometry entries still hold the slot's previous size
    uint8_t* d_bgr = nullptr;           // staging of colour (BGR) inputs, converted by k_bgr_to_gray (ingest.cu)
    size_t bgr_bytes = 0;
    // SM partition (green contexts, ctx.cu vo_partition_enable): the LK ring kernel -- persistent, 100 % of the registers of
    // every SM it runs on -- shares its SMs only with the throughput kernels before it (FAST, pyramids); the latency-bound
    // kernels after the ring (filters, triangulation, PnP) run on the rest, so those of one unit range execute WHILE the
    // other range's LK ring does
    bool part_on = false;
    bool part_auto = true;              // the first vo_batch_submit turns the partition on (8 SMs for the kernels after the ring)
    int part_helper_sms = 0, part_lk_sms = 0;
    void* part_gctx[2] = {nullptr, nullptr};            // CUgreenCtx: [0] helpers, [1] LK
    // multi-GPU record gather over NCCL (dist.cu); NCCL is dlopen'ed at vo_dist_init
    void* dist_comm = nullptr;
    int dist_rank = 0, dist_world = 1;
    cudaStream_t dist_stream = nullptr, dist_snap_stream = nullptr;     // collectives / per-post snapshots (never queued behind a collective)
    // up to VO_DIST_DEPTH posted steps outstanding.  A post only snapshots the records (device to device) into the open
    // bucket; a bucket is exchanged with ONE in-place all-gather + ONE copy to pinned memory when it holds VO_DIST_BUCKET
    // steps, or earlier when the host asks for one of its steps.
    struct DistBucket { void* d = nullptr; void* h = nullptr; cudaEvent_t done = nullptr; int fill = 0, unwaited = 0, n_units = 0; bool flushed = false; };
    struct DistStep { int bucket = 0, index = 0; };
    DistBucket dist_bk[VO_DIST_NB];
    DistStep dist_steps[2 * VO_DIST_DEPTH];
    int dist_cur = 0;
    cudaEvent_t dist_ev_read = nullptr, dist_ev_fork = nullptr;
    size_t dist_bytes = 0;
    long long dist_head = 0, dist_tail = 0;
    // mono_rotation branch (ess.cu): scratch of the essential-matrix RANSAC, allocated on first use
    void* d_ess = nullptr;
    int ess_cap = 0;
    // the same branch inside the sequence mode (vo_set_option "mono_rotation" for vo_seq_begin*, the flag
    // VO_MSEQ_MONO_ROTATION for vo_mseq_begin_ex): one scratch block per buffer unit (2 * seq_n: two frames in flight),
    // separate from d_ess, allocated at the begin call; the front graph runs it for every sequence on seq_mono_stream
    bool mono_opt = false;              // the option; a vo_seq_* sequence takes it at vo_seq_begin
    bool seq_mono = false;              // the running sequences' value
    void* d_seq_ess = nullptr;          // [seq_ess_units][seq_ess_bytes], block u = buffer unit u
    size_t seq_ess_bytes = 0;
    int seq_ess_cap = 0;                // points each block holds (the bucket grid, at most cap)
    int seq_ess_units = 0;              // blocks allocated
    cudaStream_t seq_mono_stream = nullptr;
    cudaEvent_t seq_mono_ev[2] = {nullptr, nullptr};     // fork, join
    std::vector<void*> allocs;          // everything cudaMalloc'ed for the batch state

    // ---- pinned host staging ------------------------------------------------------------------
    void* h_pinned = nullptr;
    size_t h_pinned_bytes = 0;

    // ---- LK kernel timing (CUDA events on the launching stream) -------------------------------
    std::vector<cudaEvent_t> ev_pool;   // pairs: start, stop
    size_t ev_used = 0;
    double lk_ms = 0.0;
    long long lk_n = 0;
    bool lk_timing = true;
    bool lk_use_tma = true;
    int lk_span = 0;                    // phases per LK work item: 0 = automatic (one level-solve per item when a launch has
                                        // more features than resident warps, else one item per feature-ring)
    int* d_lk_progress = nullptr;       // [units][cap] hand-over counters of the LK work items (zero between launches)
    // work queues of the persistent LK warps: one (next, dry) pair per stream that launches the kernel,
    // so launches of different streams never share a pair; a pair resets itself at the end of a launch
    int* d_lk_queue = nullptr;          // [LK_QUEUES][2]
    std::vector<cudaStream_t> lk_queue_streams;

    // ---- batched path bookkeeping -----------------------------------------------------------
    int batch_units = 0;            // units configured by vo_batch_configure
    int batch_uploaded = 0;         // units currently resident
    bool batch_detect = false;      // features come from the on-GPU FAST + stride selection
    int batch_streams = 2;          // unit ranges run concurrently by the batched path
    bool use_graphs = true;         // replay the per-range kernel sequence as a CUDA graph (no LK event timing then)
    struct CachedGraph { GraphKey key; cudaGraphExec_t exec; long long launches; };
    std::vector<CachedGraph> graphs; // invalidated when the device state is re-allocated
    std::vector<int> slot_pts;      // [batch_units] feature bound of each slot: n_pts of the unit last uploaded into it
    // One lane per submission in flight: vo_frame_batch / vo_batch_run put their unit ranges on lanes 0 and 1 (H2D of one
    // under the compute of the other), vo_batch_submit cycles through all of them, and the sequence mode solves poses on
    // lane 0 and uploads on lane 1.  A range on a lane runs FAST + pyramids on `pre`, its LK ring on `lk` and everything
    // after the ring on `post`, ordered by ev[0..3].  With the SM partition on, pre = lk = the LK partition's stream and
    // post = the helper partition's (vo_partition_enable); otherwise pre = post = a high-priority helper stream and lk =
    // side (created on first use), so the helpers' few CTAs never queue behind the other range's LK launch.
    struct Lane {
        cudaStream_t side = nullptr;                    // forked from / joined into ctx->stream
        cudaStream_t pre = nullptr, lk = nullptr, post = nullptr;
        cudaEvent_t join = nullptr, ev[4] = {};
    };
    Lane lane[VO_LANES];
    cudaEvent_t fork_ev = nullptr;
    struct Pending { int u0 = 0, n = 0; bool active = false; cudaEvent_t done = nullptr; };
    std::vector<Pending> pending;   // vo_batch_submit / vo_batch_wait
    // full outputs of a submission (what matchingFeatures / trackingFrame2Frame hand back): packed per unit on the
    // device and copied with ONE D2H per submission into pinned staging (vo_set_option "batch_outputs")
    bool batch_outputs = false;
    uint8_t* d_out = nullptr;       // [units][out_stride]  (part of the batch state)
    uint8_t* h_out = nullptr;       // pinned, [out_units][out_stride]
    size_t out_stride = 0;
    int out_per = 0, out_units = 0; // point slots per unit in a packed block (>= every resident slot's bound); units the pinned block holds
    unsigned submit_count = 0;
};

void vo_set_error(vo_ctx* ctx, const char* fmt, ...);
// levels > 0: that pyramid depth (the common depth of a run's image sizes, which their envelope w x h may exceed)
int vo_ensure_state(vo_ctx* ctx, int w, int h, int units, int levels = 0);
// geometry table entries [p0, p0 + n) = g[0 .. n), written on st (nullptr: ctx->stream) only where they change (as
// vo_write_calib)
int vo_write_geo(vo_ctx* ctx, int p0, int n, const PlaneGeom* g, cudaStream_t st = nullptr);
// the geometry of a w x h image in the allocated pyramid's levels (raw rows packed)
PlaneGeom vo_plane_geom(const vo_ctx* ctx, int w, int h);
void vo_free_state(vo_ctx* ctx);
void vo_drop_graphs(vo_ctx* ctx);
// replays the graph cached for `key` on key.s, or captures what `launch` enqueues there, caches and replays it (plain
// `launch` with the option graphs = 0).  LK event timing is off during a capture.
int vo_run_graph(vo_ctx* ctx, const GraphKey& key, const std::function<int()>& launch);
// the lanes' side streams and fork / join events (their pre / lk / post streams are filled in by the partition or on
// first use of the priority helpers)
int vo_ensure_lanes(vo_ctx* ctx);
// Calibration table entries [1 + u0, 1 + u0 + n) (buffer units u0 ..; u0 = -1 is the stage calls' entry) = c[0 .. n),
// written on ctx->stream only where they change.  The copy is queued after every batch submission still in flight, so
// it never lands under one; sequence frames in flight are the caller's to refuse or drain.
int vo_write_calib(vo_ctx* ctx, int u0, int n, const CamCalib* c);
// buffer units [u0, u0 + n): unit u0 + i from the matrices P_l + 12 * (i % n_mat), P_r + 12 * (i % n_mat)
int vo_set_calibration(vo_ctx* ctx, int u0, int n, const float* P_l, const float* P_r, int n_mat);
// Parameter table entries [1 + u0, 1 + u0 + n) = e[0 .. n), written as vo_write_calib writes its table
int vo_write_params(vo_ctx* ctx, int u0, int n, const UnitParams* e);
// the kernels' entry of a vo_params
UnitParams vo_unit_params(const vo_params& p);
// The field rules vo_create applies to a vo_params (every field but max_features and max_units): VO_E_INVALID or
// VO_E_UNSUPPORTED with vo_create's message
int vo_check_params(vo_ctx* ctx, const vo_params& p);
// vo_check_params, then the rules of a unit's or slot's own vo_params against the context's (who / what: "vo_mseq_params",
// "slot 3"): lk_win, lk_max_level and fast_nonmax equal (VO_E_UNSUPPORTED), pnp_iterations within the RANSAC scratch
// (VO_E_CAPACITY)
int vo_check_unit_params(vo_ctx* ctx, const char* who, const char* what, const vo_params& p);
int vo_drain_pending(vo_ctx* ctx);
// Entry points that overwrite the shared image planes / unit-0 buffers call this first: refused (VO_E_INVALID) while
// sequence frames or batch submissions are in flight; an idle sequence is ended (its planes are about to be reused).
int vo_partition_enable(vo_ctx* ctx, int helper_sms);       // 0 = off
void vo_partition_destroy(vo_ctx* ctx);
int vo_dist_order_after_gathers(vo_ctx* ctx, cudaStream_t st);
void vo_dist_shutdown(vo_ctx* ctx);
int vo_claim_buffers(vo_ctx* ctx, const char* who, bool allow_pending_batches = false);
// VO_E_INVALID + message while a vo_batch_submit submission has not been waited for
int vo_refuse_pending_batches(vo_ctx* ctx, const char* who);
int vo_ensure_pinned(vo_ctx* ctx, size_t bytes);
// H2D of a host image (h rows of row_bytes, pitch bytes apart) into a packed device plane on st: one 1-D copy when the
// rows are contiguous, else a 2-D copy
int vo_upload_plane(vo_ctx* ctx, uint8_t* dst, const uint8_t* src, size_t row_bytes, int h, size_t pitch, cudaStream_t st);
int vo_ensure_bgr(vo_ctx* ctx, size_t bytes);
// k_bgr_to_gray: images tab[0 .. n_img) (device table), or with d_tab == nullptr `packed` advanced by packed_stride per image,
// into gray planes img_stride_out apart; geo: the images' geometry table entries (nullptr: all w x h).  A table entry
// with data == NULL is skipped.
int vo_launch_bgr_to_gray(const vo_dimage* d_tab, const vo_dimage& packed, size_t packed_stride, uint8_t* d_gray, size_t img_stride_out,
                          int w, int h, int n_img, cudaStream_t s, const PlaneGeom* geo = nullptr);
vo_dimage vo_packed_bgr(const uint8_t* d_bgr, int w);      // the descriptor of w-pixel packed BGR rows
// VO_E_INVALID + message unless `im` can be read as an image `w` pixels wide in device memory of the context's GPU
int vo_check_dimage(vo_ctx* ctx, const char* who, const char* name, const vo_dimage* im, int w);
// caller device images h_tab[0 .. n) (pinned staging, untouched until the copy has run on st) -> raw planes
// [plane0, plane0 + n): one descriptor copy into d_ingest_tab + plane0 and one k_bgr_to_gray launch on st.  geo: the
// planes' geometry table entries (images of several sizes, each written packed from its plane's start; nullptr: all w x h)
int vo_ingest_device(vo_ctx* ctx, const vo_dimage* h_tab, int n, int plane0, cudaStream_t st, const PlaneGeom* geo = nullptr);
// a contiguous range of resident work units processed on one stream
// plane0 >= 0 overrides the image-plane base (default u0 * imgs): the sequence mode ping-pongs its per-frame buffers
// between two buffer parities while both address the same image ring.  imgs: image planes per unit (4: a stereo pair at
// t0 and t1; 2: one LK call, or one sequence's pair in the sequence mode).  max_pts: live features per unit at most
// (0 = cap), which sizes the LK launch.
// sized: the image planes hold images of several sizes; FAST and the LK ring read each one's from the geometry table.
struct View { int u0, n; cudaStream_t s; int plane0 = -1; int imgs = 4; int max_pts = 0; bool sized = false; };
// The stage runners below read unit u's parameters from par[u] (ctx->d_par, or the stage calls' entry ctx->d_par_tab
// with v.u0 = 0) and its camera from cal[u] alike.
// run pyramids + LK (ncalls chained) for the units of `v`; images must already be in d_raw/d_raw_tab
int vo_run_lk(vo_ctx* ctx, const View& v, int ncalls, const int* img_prev, const int* img_next, bool want_err, const UnitParams* par);
// sized: the planes hold images of several sizes, read from the geometry table (vo_mseq_begin_sized)
int vo_run_pyramid(vo_ctx* ctx, int plane0, int nplanes, cudaStream_t s, bool sized = false);
int vo_run_lk_ring(vo_ctx* ctx, const View& v, int ncalls, const int* img_prev, const int* img_next, bool want_err,
                   const UnitParams* par);
int vo_run_filter(vo_ctx* ctx, const View& v, bool with_ages, const UnitParams* par);
// FAST on raw plane `plane_in_unit` of each unit -> d_corners / d_ndet ; stride selection -> d_pts_in / d_npts
int vo_run_fast(vo_ctx* ctx, const View& v, int plane_in_unit, bool want_resp, const UnitParams* par);
int vo_run_select(vo_ctx* ctx, const View& v);
// triangulate pts_l/pts_r ([units][cap], counts n) -> d_X ; PnP on (d_X, pts2d) -> d_results / d_inliers.  Unit u reads
// the camera cal[u] (ctx->d_cal, or the stage calls' single entry with v.u0 = 0).
int vo_run_triangulate(vo_ctx* ctx, const View& v, const float2* pts_l, const float2* pts_r, const int* n, const CamCalib* cal,
                       float4* X4 = nullptr);
int vo_run_pnp(vo_ctx* ctx, const View& v, const float2* pts2d, const int* n, const CamCalib* cal, const UnitParams* par);
// RANSAC iterations the PnP stage sizes and runs: cv::RANSACPointSetRegistrator runs at least one (max(maxIters, 1))
inline int vo_pnp_iterations(const vo_ctx* ctx) { return ctx->p.pnp_iterations > 1 ? ctx->p.pnp_iterations : 1; }
