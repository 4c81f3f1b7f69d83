// filter.cu -- K3: ring filters + order-preserving compaction, one CTA per work unit.
//
// Replaces, bug-for-bug (SURVEY.md Appendix A items 3, 4, 7, 8):
//   deleteUnmatchFeaturesCircle()   reference src/feature.cpp:76-116
//       ages[i] += 1 for all; drop i iff any status0..3[i]==0 or any of pt0..pt3 has x<0 or y<0
//       (points0_return is NOT tested); erase from the 5 point vectors + ages, order preserved.
//   checkValidMatch(thr=0)          reference src/visualOdometry.cpp:44-61,119-120
//       int offset = max(|dx|,|dy|) (float -> int truncation); valid iff offset <= thr
//   removeInvalidPoints() x4        reference src/visualOdometry.cpp:63-77,122-125
//       compacts pL0, pL1, pR0, pR1 -- but NOT features.ages (kept at the A3 length).
// The arithmetic is compare-only; oracle restatement: oracle/ref_path.py.
#include "common.cuh"
#include "filter.h"

#define FT 1024

__global__ void __launch_bounds__(FT) k_ring_filter(const FilterArgs a)
{
    const int unit = blockIdx.x;
    const int n = a.n_pts[unit];
    const int circ_threshold = a.par[unit].circ_threshold;
    const size_t ub = (size_t)unit * a.cap;
    const float2* p0 = a.pts_in + ub;                        // L0
    const float2* p1 = a.pts_out + 0 * a.call_stride + ub;   // R0
    const float2* p2 = a.pts_out + 1 * a.call_stride + ub;   // R1
    const float2* p3 = a.pts_out + 2 * a.call_stride + ub;   // L1
    const float2* pr = a.pts_out + 3 * a.call_stride + ub;   // L0 return
    const uint8_t* s0 = a.status + 0 * a.call_stride + ub;
    const uint8_t* s1 = a.status + 1 * a.call_stride + ub;
    const uint8_t* s2 = a.status + 2 * a.call_stride + ub;
    const uint8_t* s3 = a.status + 3 * a.call_stride + ub;

    __shared__ int wcnt3[32], wcnt5[32];
    __shared__ int base3, base5;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { base3 = 0; base5 = 0; }
    __syncthreads();

    for (int c0 = 0; c0 < n; c0 += FT) {
        const int i = c0 + threadIdx.x;
        bool keep3 = false, keep5 = false;
        float2 q0, q1, q2, q3, qr;
        if (i < n) {
            q0 = p0[i]; q1 = p1[i]; q2 = p2[i]; q3 = p3[i]; qr = pr[i];
            const bool bad = (s3[i] == 0) || (q3.x < 0) || (q3.y < 0) || (s2[i] == 0) || (q2.x < 0) || (q2.y < 0) ||
                             (s1[i] == 0) || (q1.x < 0) || (q1.y < 0) || (s0[i] == 0) || (q0.x < 0) || (q0.y < 0);
            keep3 = !bad;
            if (keep3) {
                const float m = fmaxf(fabsf(q0.x - qr.x), fabsf(q0.y - qr.y));
                const int offset = (int)m;            // float -> int truncation, as the reference's `int offset`
                keep5 = !(offset > circ_threshold);
            }
        }
        const unsigned b3 = __ballot_sync(0xffffffffu, keep3);
        const unsigned b5 = __ballot_sync(0xffffffffu, keep5);
        if (lane == 0) { wcnt3[warp] = __popc(b3); wcnt5[warp] = __popc(b5); }
        __syncthreads();
        int off3 = base3, off5 = base5;
        for (int w = 0; w < warp; w++) { off3 += wcnt3[w]; off5 += wcnt5[w]; }
        const unsigned lt = (1u << lane) - 1u;
        if (keep3) {
            const int o = off3 + __popc(b3 & lt);
            a.kept5[0 * a.call_stride + ub + o] = q0;
            a.kept5[1 * a.call_stride + ub + o] = q1;
            a.kept5[2 * a.call_stride + ub + o] = q3;   // L1
            a.kept5[3 * a.call_stride + ub + o] = q2;   // R1
            a.kept5[4 * a.call_stride + ub + o] = qr;
            a.idx3[ub + o] = i;
            if (a.ages_in) a.ages_out[ub + o] = a.ages_in[ub + i] + 1;
        }
        if (keep5) {
            const int o = off5 + __popc(b5 & lt);
            a.valid4[0 * a.call_stride + ub + o] = q0;   // L0
            a.valid4[1 * a.call_stride + ub + o] = q1;   // R0
            a.valid4[2 * a.call_stride + ub + o] = q3;   // L1
            a.valid4[3 * a.call_stride + ub + o] = q2;   // R1
            a.idx5[ub + o] = i;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int t3 = 0, t5 = 0;
            for (int w = 0; w < FT / 32; w++) { t3 += wcnt3[w]; t5 += wcnt5[w]; }
            base3 += t3; base5 += t5;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { a.n3[unit] = base3; a.n5[unit] = base5; }
}

cudaError_t vo_launch_ring_filter(const FilterArgs& a, int n_units, cudaStream_t stream)
{
    if (n_units <= 0) return cudaSuccess;
    k_ring_filter<<<n_units, FT, 0, stream>>>(a);
    return cudaGetLastError();
}
