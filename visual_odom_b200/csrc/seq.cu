// seq.cu -- streaming sequence mode (SURVEY.md section 8f row N1): the reference's main loop state
// (src/main.cpp:87-92,123-181: currentVOFeatures, the previous stereo pair, `translation`) kept resident
// on the device, so one vo_seq_push() uploads only the NEW stereo pair, builds only its two pyramids
// (the previous pair's pyramids are reused as t0) and runs matchingFeatures() -> triangulation ->
// trackingFrame2Frame() without a host round trip.
//
// The glue between the OpenCV-backed stages is the reference's own, restated bug-for-bug on the device:
//   appendNewFeatures   src/feature.cpp:255-262  (refill while fewer than vo_params.refill_threshold features, 2000 in the
//        reference: always at one feature per bucket, in practice)
//   bucketingFeatures   src/feature.cpp:206-253 + Bucket::add_feature src/bucket.cpp:14-45
//        (nh+1)*(nw+1) cells of rows / bucket_rows_divisor pixels addressed with row stride nw (aliasing + duplicated
//        read-back), ages >= bucket_age_threshold refused, features_per_bucket slots per cell of which a full cell
//        overwrites slot 0 (at one slot: the LAST admitted feature in input order wins)
//   the ages / points length skew after the circular check (src/visualOdometry.cpp:122-127): point i is
//        paired with ages[i] even though the ages vector is longer and shifted.
//
// Each kernel serves n_seq independent sequences in one launch (blockIdx.y = sequence, strides in SeqArgs); the
// single-sequence mode launches them with n_seq = 1.
#include "common.cuh"
#include "seq.h"
#include "pose_math.cuh"
#include <climits>

__global__ void __launch_bounds__(1024) k_seq_append(const float2* __restrict__ corners, const int* __restrict__ n_det,
                                                     int corner_cap, float2* feat_pts, int* feat_ages, int* cnt, int feat_cap,
                                                     const UnitParams* __restrict__ par, int* err, const int* __restrict__ live)
{
    const int q = blockIdx.y;
    corners += (size_t)q * corner_cap; n_det += q; feat_pts += (size_t)q * feat_cap; feat_ages += (size_t)q * feat_cap;
    cnt += 2 * q; err += q;
    // the error bits are per frame: this is the first glue kernel of a frame's front stage, it clears the frame's word
    if (threadIdx.x == 0) *err = 0;
    __syncthreads();
    if (!live[q]) return;                              // retired: the state stays as it is
    const int n_pts = cnt[0], n_ages = cnt[1];
    // `if (currentVOFeatures.size() < 2000)`: no refill leaves the FeatureSet as it is (n_det still counts the corners)
    if (n_pts >= par[q].refill_threshold) return;
    int m = *n_det;
    if (m > corner_cap) { m = corner_cap; if (threadIdx.x == 0) atomicOr(err, 1); }
    if (n_pts + m > feat_cap || n_ages + m > feat_cap) { m = min(feat_cap - n_pts, feat_cap - n_ages); if (m < 0) m = 0; if (threadIdx.x == 0) atomicOr(err, 2); }
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        feat_pts[n_pts + i] = corners[i];
        feat_ages[n_ages + i] = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) { cnt[0] = n_pts + m; cnt[1] = n_ages + m; }
}

// bucketingFeatures() with Bucket(max_size = k): cells of bucket_size = rows / divisor pixels, features aged
// >= age_threshold refused.  Bucket::add_feature's "replace youngest" loop compares the incoming age with itself, so a
// full bucket always overwrites slot 0: with a_1 .. a_c the features admitted to a cell in input order, the cell reads
// back as a_1 .. a_c when c <= k and as a_c, a_2, .. a_k when c > k.  So a cell needs its k smallest admitted indices
// and its largest one.  Both are order-free: atomicMax keeps the largest, and the k sorted slots of the cell take the k
// smallest through a cascade of atomicMin (a slot keeps the smaller of what it holds and what comes in and passes the
// larger one on, so slot s ends up with the (s + 1)-th smallest index whatever order the threads run in).  The number of
// filled slots is min(c, k), and c > k exactly when the cell is full and its largest index is not its k-th smallest.
// Scratch per sequence: last[nb] | first[nb][k].  At k = 1 every non-empty cell reads back its last admitted feature.
// (One block per SM: with k, the gate and the divisor read from the sequence's parameter entry, the default bound of two
// blocks per SM leaves 32 registers and spills; a launch has one block per sequence, far fewer than the SMs.)
__global__ void __launch_bounds__(1024, 1) k_seq_bucket(const float2* __restrict__ feat_pts, const int* __restrict__ feat_ages,
                                                     int feat_cap, const int* __restrict__ cnt, int rows, int cols,
                                                     const UnitParams* __restrict__ par, int* bucket /* scratch */, size_t nb_cap,
                                                     float2* out_pts, int* out_ages, int* out_n, int out_cap, int* err,
                                                     const int* __restrict__ live, const PlaneGeom* __restrict__ geo, int geo_stride)
{
    const int q = blockIdx.y;
    if (geo) {             // the sequence's own grid: the stride-nw aliasing below depends on nw
        rows = geo[q * geo_stride].h[0]; cols = geo[q * geo_stride].w[0];
    }
    const int divisor = par[q].bucket_rows_divisor, k = par[q].features_per_bucket, age_threshold = par[q].bucket_age_threshold;
    const int bucket_size = rows / divisor;
    feat_pts += (size_t)q * feat_cap; feat_ages += (size_t)q * feat_cap; cnt += 2 * q; bucket += (size_t)q * nb_cap;
    out_pts += (size_t)q * out_cap; out_ages += (size_t)q * out_cap; out_n += q; err += q;
    if (!live[q]) { if (threadIdx.x == 0) *out_n = 0; return; }        // retired: no features, so no work downstream
    // a zero bucket size and a grid above the scratch are refused by the begin / start calls
    if (bucket_size <= 0) { if (threadIdx.x == 0) { atomicOr(err, 4); *out_n = 0; } return; }
    const int nh = rows / bucket_size, nw = cols / bucket_size;
    const int nb = (nh + 1) * (nw + 1);
    if ((size_t)nb * (k + 1) > nb_cap) { if (threadIdx.x == 0) { atomicOr(err, 4); *out_n = 0; } return; }
    int* last = bucket;
    int* first = bucket + nb;
    for (int b = threadIdx.x; b < nb; b += blockDim.x) last[b] = -1;
    for (int j = threadIdx.x; j < nb * k; j += blockDim.x) first[j] = INT_MAX;
    __syncthreads();
    const int n = cnt[0];
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (feat_ages[i] < age_threshold) {                              // Bucket::add_feature: age < age_threshold
            const float2 p = feat_pts[i];
            const int bh = (int)(p.y / (float)bucket_size), bw = (int)(p.x / (float)bucket_size);
            const int idx = bh * nw + bw;                                // row stride nw, not nw + 1
            if (idx >= 0 && idx < nb) {
                atomicMax(&last[idx], i);
                int* f = first + (size_t)idx * k;
                // slots only shrink: a k-th smallest already below i (even as read before the latest update) keeps i out
                if (__ldcg(f + k - 1) > i) {
                    int v = i;
                    for (int s = 0; s < k; s++) {
                        const int o = atomicMin(f + s, v);
                        if (o == INT_MAX) break;                         // v took an empty slot
                        v = max(o, v);                                   // the larger one moves on
                    }
                }
            } else {
                atomicOr(err, 8);                                        // outside the image: undefined behaviour in the reference
            }
        }
    }
    __syncthreads();
    auto filled = [&](int b) {                                           // min(c, k): the filled slots are a prefix
        const int* f = first + (size_t)b * k;
        int m = 0;
        while (m < k && f[m] != INT_MAX) m++;
        return m;
    };
    // ordered read-back (same aliased addressing as the reference): cell sequence q = h * (nw + 1) + w, h <= nh, w <= nw.
    // Each thread takes a contiguous chunk of q, a block-wide exclusive scan of the chunk counts gives its output offset.
    __shared__ int s_cnt[1024];
    const int per = (nb + blockDim.x - 1) / blockDim.x;
    const int q0 = threadIdx.x * per, q1 = min(nb, q0 + per);
    int mine = 0;
    for (int q = q0; q < q1; q++) {
        const int h = q / (nw + 1), w = q - h * (nw + 1);
        mine += filled(h * nw + w);
    }
    s_cnt[threadIdx.x] = mine;
    __syncthreads();
    for (int d = 1; d < (int)blockDim.x; d <<= 1) {           // Hillis-Steele inclusive scan
        const int v = threadIdx.x >= d ? s_cnt[threadIdx.x - d] : 0;
        __syncthreads();
        s_cnt[threadIdx.x] += v;
        __syncthreads();
    }
    int m = s_cnt[threadIdx.x] - mine;
    for (int q = q0; q < q1; q++) {
        const int h = q / (nw + 1), w = q - h * (nw + 1), b = h * nw + w;
        const int* f = first + (size_t)b * k;
        const int c = filled(b);
        const bool over = c == k && last[b] != f[k - 1];              // more than k admitted: a_c sits in slot 0
        for (int s = 0; s < c; s++, m++) {
            const int j = s == 0 && over ? last[b] : f[s];
            if (m < out_cap) { out_pts[m] = feat_pts[j]; out_ages[m] = feat_ages[j]; }
        }
    }
    if (threadIdx.x == blockDim.x - 1) {
        const int total = s_cnt[threadIdx.x];
        if (total > out_cap) atomicOr(err, 4);                           // the begin / start calls keep the bound within out_cap
        *out_n = min(total, out_cap);
    }
}

// after the circular check: currentVOFeatures.points = pointsLeft_t1 (A5 survivors), the ages keep their A3 length
// (src/visualOdometry.cpp:122-127).  Runs before the pose solve, so the next frame's front half can start under it.
__global__ void __launch_bounds__(256) k_seq_carry(const float2* __restrict__ valid_l1, const int* __restrict__ n5,
                                                   const int* __restrict__ ages_out, const int* __restrict__ n3,
                                                   int cap, float2* feat_pts, int* feat_ages, int feat_cap, int* cnt,
                                                   const int* __restrict__ live)
{
    const int q = blockIdx.y;
    if (!live[q]) return;
    valid_l1 += (size_t)q * cap; n5 += q; ages_out += (size_t)q * cap; n3 += q;
    feat_pts += (size_t)q * feat_cap; feat_ages += (size_t)q * feat_cap; cnt += 2 * q;
    const int np = *n5, na = *n3;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(np, na); i += gridDim.x * blockDim.x) {
        if (i < np) feat_pts[i] = valid_l1[i];
        if (i < na) feat_ages[i] = ages_out[i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { cnt[0] = np; cnt[1] = na; }
}

// after the pose solve: `translation` carries the solved tvec to the next frame's solve; counts into the result record
__global__ void k_seq_finish(vo_unit_result_dev* res, double* tprev_next, const double* __restrict__ tprev_cur,
                             const int* __restrict__ n_feat, const int* __restrict__ n_det, const int* __restrict__ n3,
                             const int* __restrict__ n5, const int* __restrict__ err, int* err_out, const int* __restrict__ live)
{
    const int q = blockIdx.y;
    res += q; tprev_next += 3 * q; tprev_cur += 3 * q; n_feat += q; n_det += q; n3 += q; n5 += q; err += q; err_out += q;
    if (!live[q]) {                                    // retired: the translation stays frozen in both buffer slots
        if (threadIdx.x < 3) tprev_next[threadIdx.x] = tprev_cur[threadIdx.x];
        return;
    }
    if (threadIdx.x == 0) {
        for (int k = 0; k < 3; k++) tprev_next[k] = res->tvec[k];
        res->n_features = *n_feat; res->n_detected = *n_det; res->n_tracked = *n3; res->n_valid = *n5;
        if (err_out != err) *err_out = *err;
    }
}

// trackingFrame2Frame(mono_rotation = true) (src/visualOdometry.cpp:146-157,186-189): `rotation` comes from recoverPose,
// the PnP supplies only `translation`.  Runs after k_seq_finish, so the translation carry is the PnP's as without the branch.
// Sequence q's result is ess_stride bytes after sequence q - 1's.
__global__ void k_seq_mono(vo_unit_result_dev* res, const EssResult* __restrict__ ess, size_t ess_stride, const int* __restrict__ live)
{
    const int q = blockIdx.y;
    if (!live[q]) return;
    res += q;
    ess = (const EssResult*)((const char*)ess + (size_t)q * ess_stride);
    const int k = threadIdx.x;
    if (k < 9) res->R[k] = ess->status == ESS_OK ? ess->R[k] : (k % 4 == 0 ? 1.0 : 0.0);
}

// vo_mseq_wait_device (K7): one block per sequence retires the oldest submission into the caller's buffers -- what
// seq_wait does on the host from the pinned copies, and the point lists, points3D and inliers it leaves in the units.
// Thread 0 writes the status / record / mono result and integrates frame_pose (main.cpp:196-208: a frame is integrated
// when its PnP ran (VO_OK or no model) and, with mono_rotation, the essential branch did not abort); the block copies the
// lists.  Sequences are independent, so the launch is one grid however many of them there are.
__global__ void __launch_bounds__(256) k_seq_collect(const CollectArgs a)
{
    const int q = blockIdx.x, mode = a.mode[q];
    const vo_unit_result_dev* res = a.res + q;
    const EssResult* ess = a.ess ? (const EssResult*)((const char*)a.ess + (size_t)q * a.ess_stride) : nullptr;
    double* pose = a.pose + 16 * (size_t)q;
    const int nv = mode == 1 ? min(res->n_valid, a.pts_cap) : 0;
    const int ni = mode == 1 ? min(res->n_inliers, a.pts_cap) : 0;
    if (threadIdx.x == 0) {
        int status = mode == SEQ_STARTED ? VO_MSEQ_STARTED : VO_MSEQ_RETIRED;
        vo_unit_result_dev r;
        memset(&r, 0, sizeof(r));
        vo_mono_result m;
        memset(&m, 0, sizeof(m));
        if (mode == 1) {
            r = *res;
            const bool mono_ok = !ess || ess->status == ESS_OK;
            if ((r.pnp_status == VO_OK || r.pnp_status == VO_PNP_NO_MODEL) && mono_ok) vo_pose_step_dev(pose, r.R, r.tvec);
            if (ess) {
                m.status = mono_ok ? VO_OK : VO_E_TOO_FEW_POINTS;
                m.n_inliers = ess->n_inliers; m.ransac_iters = ess->iters; m.n_good = ess->n_good;
                for (int k = 0; k < 9; k++) m.R[k] = ess->R[k];
                for (int k = 0; k < 3; k++) m.t[k] = ess->t[k];
            }
            // bit 8 (a tracked point outside the bucket grid) is not an error, as in seq_wait
            status = (a.err[q] & ~8) ? VO_E_CAPACITY : VO_OK;
        } else if (mode == SEQ_STARTED) {              // the new sequence's frame_pose starts here (main.cpp:90)
            for (int i = 0; i < 16; i++) pose[i] = i % 5 == 0 ? 1.0 : 0.0;
        }
        if (a.status) a.status[q] = status;
        if (a.records) a.records[q] = r;
        if (a.mono) a.mono[q] = m;
        if (a.pose_out)
            for (int i = 0; i < 16; i++) a.pose_out[16 * (size_t)q + i] = pose[i];
    }
    const size_t src = (size_t)q * a.cap, dst = (size_t)q * a.pts_cap;
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
        if (a.pts4)
            for (int k = 0; k < 4; k++) a.pts4[(4 * (size_t)q + k) * a.pts_cap + i] = a.valid4[k * a.plane_stride + src + i];
        if (a.points3d) a.points3d[dst + i] = a.X[src + i];
        if (a.mask_out) a.mask_out[dst + i] = a.ess_mask[(size_t)q * a.ess_stride + i];
    }
    if (a.inliers_out)
        for (int i = threadIdx.x; i < ni; i += blockDim.x) a.inliers_out[dst + i] = a.inliers[src + i];
}

int vo_launch_seq_collect(const CollectArgs& a, int n_seq, cudaStream_t s)
{
    k_seq_collect<<<n_seq, 256, 0, s>>>(a);
    return 1;
}

int vo_launch_seq_append(const SeqArgs& a, int n_seq, cudaStream_t s)
{
    k_seq_append<<<dim3(1, n_seq), 1024, 0, s>>>(a.corners, a.n_det, a.corner_cap, a.feat_pts, a.feat_ages, a.cnt, a.feat_cap,
                                                 a.par, a.err, a.live);
    return 1;
}
int vo_launch_seq_bucket(const SeqArgs& a, int n_seq, cudaStream_t s)
{
    k_seq_bucket<<<dim3(1, n_seq), 1024, 0, s>>>(a.feat_pts, a.feat_ages, a.feat_cap, a.cnt, a.rows, a.cols, a.par, a.bucket, a.bucket_cap, a.out_pts, a.out_ages, a.out_n, a.out_cap, a.err, a.live,
                                                 a.geo, a.geo_stride);
    return 1;
}
int vo_launch_seq_carry(const SeqArgs& a, int n_seq, cudaStream_t s)
{
    k_seq_carry<<<dim3(8, n_seq), 256, 0, s>>>(a.valid_l1, a.n5, a.ages_out, a.n3, a.out_cap, a.feat_pts, a.feat_ages, a.feat_cap,
                                               a.cnt, a.live);
    return 1;
}
int vo_launch_seq_finish(const SeqArgs& a, int n_seq, cudaStream_t s)
{
    k_seq_finish<<<dim3(1, n_seq), 32, 0, s>>>(a.res, a.tprev, a.tprev_cur, a.out_n, a.n_det, a.n3, a.n5, a.err, a.err_out, a.live);
    return 1;
}
int vo_launch_seq_mono(const SeqArgs& a, const EssResult* ess, size_t ess_stride, int n_seq, cudaStream_t s)
{
    k_seq_mono<<<dim3(1, n_seq), 32, 0, s>>>(a.res, ess, ess_stride, a.live);
    return 1;
}
