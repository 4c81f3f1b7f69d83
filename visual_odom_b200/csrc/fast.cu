// fast.cu -- K4: FAST-9/16 corner detector with shared-memory 3x3 non-max suppression and
// raster-ordered compaction (+ the even-stride feature selection used by the batched path).
//
// Replaces cv::FAST(image, keypoints, 20, true) + KeyPoint::convert as called by
// featureDetectionFast(), reference src/feature.cpp:39-47.  Exact arithmetic only; restated in
// oracle/fast_ref.c which is pinned list-exact (coordinates, raster order, response) against cv2.
//
//   k_fast_score   one thread per pixel: 16-pixel Bresenham ring, corner iff >= 9 contiguous ring
//                  pixels are all > p+t or all < p-t; score = max(t, max_arc min(p-r), max_arc
//                  min(r-p)) - 1 (cornerScore<16>), 0 for non-corners / the 3-pixel border.
//                  Without non-max suppression every corner is marked 1 instead (a score can be 0).
//   k_fast_nms_row one CTA per image row: the three score rows are staged in shared memory, a corner
//                  survives iff its score is strictly greater than its 8 neighbours; survivors are
//                  compacted in x order into a per-row list (ballot + running offset).
//   k_fast_scan    one CTA per unit: exclusive scan of the per-row counts -> raster offsets, total.
//   k_fast_gather  per row: copies the row list to its raster position as (x, y) floats; response =
//                  score with non-max suppression, 0 without (as cv::FAST).
//   k_select_stride  idx_i = i*(M-1)/(N-1): the benchmark's feature selection (SURVEY.md 8d).
// All HBM-bound byte work (1 B/px read, 1 B/px score write+read, 8 B/corner out).
#include "common.cuh"
#include "fast.h"

__global__ void __launch_bounds__(256) k_fast_score(const uint8_t* const* __restrict__ img_tab, int img_stride_idx,
                                                    int w, int h, int pitch, int threshold, int nonmax,
                                                    uint8_t* __restrict__ score, size_t score_plane)
{
    // the 16-pixel Bresenham ring, compile-time: the unrolled loop below folds the offsets into immediates
    constexpr int ring_dx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    constexpr int ring_dy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    const int unit = blockIdx.z;
    const uint8_t* __restrict__ img = img_tab[unit * img_stride_idx];
    uint8_t* __restrict__ sc = score + (size_t)unit * score_plane;
    const int x = blockIdx.x * 32 + (threadIdx.x & 31);
    const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= w || y >= h) return;
    int result = 0;
    if (x >= 3 && x < w - 3 && y >= 3 && y < h - 3) {
        const uint8_t* p = img + (size_t)y * pitch + x;
        const int v = p[0];
        // The differences |p - r| <= 255 are exact in float and so are their minima / maxima.  The network is kept in float
        // because NVVM's -O3 code for compute_90 computes wrong scores from the same network in int (checked pixel for pixel
        // against the host on an H100, CUDA 12.9); the float form matches the host on every pixel.
        float d[16];
        unsigned hi = 0, lo = 0;
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const int r = p[ring_dy[k] * pitch + ring_dx[k]];
            d[k] = (float)(v - r);
            hi |= (unsigned)(r > v + threshold) << k;
            lo |= (unsigned)(r < v - threshold) << k;
        }
        // >= 9 contiguous set bits on the 16-cycle
        unsigned mh = hi | (hi << 16), ml = lo | (lo << 16);
        mh &= mh >> 1; mh &= mh >> 2; mh &= mh >> 4; mh &= mh >> 1;
        ml &= ml >> 1; ml &= ml >> 2; ml &= ml >> 4; ml &= ml >> 1;
        if (mh | ml) {
            // sliding min / max over all 16 arcs of length 9 by doubling
            float mn[16], mx[16];
#pragma unroll
            for (int k = 0; k < 16; k++) { mn[k] = fminf(d[k], d[(k + 1) & 15]); mx[k] = fmaxf(d[k], d[(k + 1) & 15]); }
            float mn4[16], mx4[16];
#pragma unroll
            for (int k = 0; k < 16; k++) { mn4[k] = fminf(mn[k], mn[(k + 2) & 15]); mx4[k] = fmaxf(mx[k], mx[(k + 2) & 15]); }
            float A = -1000.f, B = 1000.f;
#pragma unroll
            for (int k = 0; k < 16; k++) {
                const float a8 = fminf(mn4[k], mn4[(k + 4) & 15]);
                const float b8 = fmaxf(mx4[k], mx4[(k + 4) & 15]);
                A = fmaxf(A, fminf(a8, d[(k + 8) & 15]));
                B = fminf(B, fmaxf(b8, d[(k + 8) & 15]));
            }
            result = max(threshold, (int)fmaxf(A, -B)) - 1;
            // Without non-max suppression the map only marks the corners (cv::FAST reports response 0): a corner's
            // score is 0 at threshold 0 when its best arc is one level beyond the centre, so the score cannot be the mark.
            if (!nonmax) result = 1;
        }
    }
    sc[(size_t)y * w + x] = (uint8_t)result;
}

#define NMS_T 256
#define NMS_NC 8                 // chunks of NMS_T pixels handled per pass: one pass covers rows up to 2048 pixels
__global__ void __launch_bounds__(NMS_T) k_fast_nms_row(const uint8_t* __restrict__ score, size_t score_plane, int w, int h,
                                                        int nonmax, uint16_t* __restrict__ rowbuf, int rowcap,
                                                        int* __restrict__ rowcount)
{
    const int y = blockIdx.x, unit = blockIdx.y;
    const uint8_t* __restrict__ sc = score + (size_t)unit * score_plane;
    uint16_t* __restrict__ out = rowbuf + ((size_t)unit * h + y) * rowcap;
    __shared__ uint8_t rows[3][NMS_T * NMS_NC + 2];
    __shared__ int wcnt[NMS_NC * (NMS_T / 32)];         // survivors per (chunk, warp), then their exclusive prefix
    __shared__ int base;
    if (y < 3 || y >= h - 3) {                     // border rows hold no corners
        if (threadIdx.x == 0) rowcount[unit * h + y] = 0;
        return;
    }
    if (threadIdx.x == 0) base = 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NW = NMS_T / 32, SPAN = NMS_T * NMS_NC;
    for (int x0 = 0; x0 < w; x0 += SPAN) {
        // stage the three score rows (with a 1-pixel halo) in shared memory: the whole pass at once
        for (int i = threadIdx.x; i < SPAN + 2; i += NMS_T) {
            const int x = x0 - 1 + i;
            const bool in = (x >= 0 && x < w);
            rows[0][i] = in ? sc[(size_t)(y - 1) * w + x] : 0;
            rows[1][i] = in ? sc[(size_t)y * w + x] : 0;
            rows[2][i] = in ? sc[(size_t)(y + 1) * w + x] : 0;
        }
        __syncthreads();
        unsigned bal[NMS_NC];
#pragma unroll
        for (int c = 0; c < NMS_NC; c++) {
            const int x = x0 + c * NMS_T + threadIdx.x, i = c * NMS_T + threadIdx.x + 1;
            bool keep = false;
            if (x < w) {
                const int s = rows[1][i];
                if (s > 0) {
                    keep = !nonmax ||
                           (s > rows[1][i - 1] && s > rows[1][i + 1] && s > rows[0][i - 1] && s > rows[0][i] &&
                            s > rows[0][i + 1] && s > rows[2][i - 1] && s > rows[2][i] && s > rows[2][i + 1]);
                }
            }
            bal[c] = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) wcnt[c * NW + warp] = __popc(bal[c]);
        }
        __syncthreads();
        // exclusive prefix over the (chunk, warp) counts in x order: 64 entries, two warps
        int carry_total = 0;
        if (threadIdx.x < NMS_NC * NW) {
            const int v = wcnt[threadIdx.x];
            int incl = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += o;
            }
            carry_total = incl;                     // lane 31 of each of the two warps holds its warp's total
            wcnt[threadIdx.x] = incl - v;
        }
        __shared__ int w0_total, pass_total;
        if (threadIdx.x == 31) w0_total = carry_total;
        __syncthreads();
        if (threadIdx.x >= 32 && threadIdx.x < NMS_NC * NW) wcnt[threadIdx.x] += w0_total;
        if (threadIdx.x == NMS_NC * NW - 1) pass_total = carry_total + w0_total;
        __syncthreads();
        const int b0 = base;
#pragma unroll
        for (int c = 0; c < NMS_NC; c++) {
            if ((bal[c] >> lane) & 1u) {
                const int o = b0 + wcnt[c * NW + warp] + __popc(bal[c] & ((1u << lane) - 1u));
                if (o < rowcap) out[o] = (uint16_t)(x0 + c * NMS_T + threadIdx.x);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) base = b0 + pass_total;
        __syncthreads();
    }
    if (threadIdx.x == 0) rowcount[unit * h + y] = base < rowcap ? base : rowcap;
}

__global__ void __launch_bounds__(1024) k_fast_scan(const int* __restrict__ rowcount, int h, int* __restrict__ rowoff,
                                                    int* __restrict__ n_det)
{
    const int unit = blockIdx.x;
    const int* rc = rowcount + unit * h;
    int* ro = rowoff + unit * h;
    __shared__ int wsum[32];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int y0 = 0; y0 < h; y0 += 1024) {
        const int y = y0 + threadIdx.x;
        int v = (y < h) ? rc[y] : 0;
        int incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int o = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += o;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        int woff = carry;
        for (int k = 0; k < warp; k++) woff += wsum[k];
        if (y < h) ro[y] = woff + incl - v;
        __syncthreads();
        if (threadIdx.x == 0) {
            int t = 0;
            for (int k = 0; k < 32; k++) t += wsum[k];
            carry += t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) n_det[unit] = carry;
}

__global__ void __launch_bounds__(128) k_fast_gather(const uint16_t* __restrict__ rowbuf, int rowcap,
                                                     const int* __restrict__ rowcount, const int* __restrict__ rowoff,
                                                     int h, const uint8_t* __restrict__ score, size_t score_plane, int w,
                                                     int nonmax, float2* __restrict__ out, float* __restrict__ resp, int cap)
{
    const int y = blockIdx.x, unit = blockIdx.y;
    const int n = rowcount[unit * h + y], off = rowoff[unit * h + y];
    const uint16_t* src = rowbuf + ((size_t)unit * h + y) * rowcap;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int o = off + i;
        if (o < cap) {
            const int x = src[i];
            out[(size_t)unit * cap + o] = make_float2((float)x, (float)y);
            if (resp)        // without non-max suppression the map holds a mark, not a score: response 0, as cv::FAST
                resp[(size_t)unit * cap + o] = nonmax ? (float)score[(size_t)unit * score_plane + (size_t)y * w + x] : 0.f;
        }
    }
}

// N features by even stride over the raster-ordered corner list (integer form of
// linspace(0, M-1, N).astype(int)); n_pts = min(N, M).
__global__ void k_select_stride(const float2* __restrict__ corners, int corner_cap, const int* __restrict__ n_det,
                                const int* __restrict__ want, float2* __restrict__ pts, int cap, int* __restrict__ n_pts)
{
    const int unit = blockIdx.y;
    int m = n_det[unit];
    if (m > corner_cap) m = corner_cap;
    int n = want[unit];
    if (n > cap) n = cap;
    if (n > m) n = m;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) n_pts[unit] = n;
    if (i >= n) return;
    const long idx = (n > 1) ? ((long)i * (m - 1)) / (n - 1) : 0;
    pts[(size_t)unit * cap + i] = corners[(size_t)unit * corner_cap + idx];
}

int vo_launch_fast(const FastArgs& a, cudaStream_t stream)
{
    dim3 g1((a.w + 31) / 32, (a.h + 7) / 8, a.n_units);
    k_fast_score<<<g1, 256, 0, stream>>>(a.img_tab, a.img_stride_idx, a.w, a.h, a.pitch, a.threshold, a.nonmax, a.score,
                                          a.score_plane);
    dim3 g2(a.h, a.n_units);
    k_fast_nms_row<<<g2, NMS_T, 0, stream>>>(a.score, a.score_plane, a.w, a.h, a.nonmax, a.rowbuf, a.rowcap, a.rowcount);
    k_fast_scan<<<a.n_units, 1024, 0, stream>>>(a.rowcount, a.h, a.rowoff, a.n_det);
    k_fast_gather<<<g2, 128, 0, stream>>>(a.rowbuf, a.rowcap, a.rowcount, a.rowoff, a.h, a.score, a.score_plane, a.w,
                                           a.nonmax, a.corners, a.resp, a.corner_cap);
    return 4;
}

int vo_launch_select(const float2* corners, int corner_cap, const int* n_det, const int* want, float2* pts, int cap,
                     int* n_pts, int n_units, cudaStream_t stream)
{
    dim3 g((cap + 255) / 256, n_units);
    k_select_stride<<<g, 256, 0, stream>>>(corners, corner_cap, n_det, want, pts, cap, n_pts);
    return 1;
}
