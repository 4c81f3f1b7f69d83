// lk_win.cu -- K2b: the LK ring at any square window from 3x3 to 32x32 (vo_params.lk_win other than 21).
//
// Same work and the same bits as k_lk_ring (lk_ring.cu), which stays the kernel for the reference's 21x21 window: the
// ncalls chained calcOpticalFlowPyrLK calls of one feature, restated in oracle/lk_ref.c (lk_track), which takes the window
// as a parameter and is pinned bit for bit against cv2 4.13.0 at every window from 3 to 32.  This kernel takes the window
// at run time, so one instance serves every width:
//   * fixed-point bilinear patches (weights cvRound(w*2^14), DESCALE by 9 / 14), half = (W - 1) * 0.5f, the
//     out-of-image tests at -W
//   * OpenCV's float32 chains: with nsimd = (W / 8) * 8 the columns x < nsimd go to SIMD lane x & 3 and the columns
//     nsimd.. to a scalar tail, rows outermost; A's addends are products of the gradients, b's are float(int pair sum)
//     of columns (x, x + 4); each total is tail + ((c0 + c2) + (c1 + c3))
//   * minEig / (2 W^2), err = sum |diff| / (32 W^2) (sum |diff| <= 1024 * 8160 < 2^24: an exact integer), the level-0
//     final re-check.
// Every sum is the faithful float chain; there is no exact-integer fast path.
//
// Parallelisation: one warp per feature-ring, taken from the launch's work queue (queue[0] = next feature, queue[1] = warps
// that ran dry; the last warp to retire resets both, the contract k_lk_ring keeps).  One work item is a whole ring:
// LkArgs::span and progress are not used (progress stays all zero), and the windows are read with plain loads from the
// padded planes (img_base / der_base / pitch / plane), never with TMA, so the lk_span option does not apply.
// The padding of VO_PAD = 32 pixels covers every read: a window starts at -W <= ipx <= w - 1 and reads columns
// ipx .. ipx + W, so reads stay in [-32, w + 31] (rows likewise).
//
// Work mapping: lane x owns window column x (lanes >= W idle) and walks its rows, so the two taps of a row are loaded once
// and serve as the bottom taps of one pixel and the top taps of the next.  The patch (I x32, Ix, Iy) and each iteration's
// residuals go to the warp's shared memory; one RUNNER lane per (quantity, chain) then forms the chain's addends from them
// and adds them strictly in order.
#include "common.cuh"
#include "lk_ring.h"

#define FULL 0xffffffffu
#define W_BITS 14
#define LKW_MAX 32
#define LKW_WARPS_PER_CTA 4
#define LKW_CTAS_PER_SM 6

namespace {

struct WinSmem {
    uint32_t grad[LKW_MAX * LKW_MAX];       // (Ix & 0xffff) | Iy << 16 of pixel (y, x) at y * LKW_MAX + x       4096
    int16_t ival[LKW_MAX * LKW_MAX];        // the patch intensities (x32)                                          2048
    int16_t diff[LKW_MAX * LKW_MAX];        // one iteration's residuals J - I                                      2048
};

__device__ __forceinline__ void bilinear_weights(float a, float b, int& w00, int& w01, int& w10, int& w11)
{
    w00 = __float2int_rn((1.f - a) * (1.f - b) * (float)(1 << W_BITS));
    w01 = __float2int_rn(a * (1.f - b) * (float)(1 << W_BITS));
    w10 = __float2int_rn((1.f - a) * b * (float)(1 << W_BITS));
    w11 = (1 << W_BITS) - w00 - w01 - w10;
}

__device__ __forceinline__ int gx(uint32_t g) { return (int)(short)(g & 0xffff); }
__device__ __forceinline__ int gy(uint32_t g) { return (int)g >> 16; }

// totals of the quantities held by the runner lanes 5q..5q+4 (chains 0..3, tail): tail + ((c0 + c2) + (c1 + c3)), in lane 5q
__device__ __forceinline__ float combine_chains(float acc)
{
    const float t1 = __fadd_rn(acc, __shfl_down_sync(FULL, acc, 2));     // lane 5q: c0 + c2, lane 5q+1: c1 + c3
    const float t2 = __fadd_rn(t1, __shfl_down_sync(FULL, t1, 1));       // lane 5q: (c0 + c2) + (c1 + c3)
    return __fadd_rn(__shfl_down_sync(FULL, acc, 4), t2);                // + tail
}

// One A chain: quantity qa (0: Ix*Ix, 1: Ix*Iy, 2: Iy*Iy), chain c (0..3: SIMD lane c, 4: the tail)
__device__ float run_a_chain(const WinSmem& sm, int win, int nsimd, int qa, int c)
{
    float acc = 0.f;
    for (int y = 0; y < win; y++) {
        const uint32_t* g = sm.grad + y * LKW_MAX;
        const int x0 = c < 4 ? c : nsimd, x1 = c < 4 ? nsimd : win, dx = c < 4 ? 4 : 1;
        for (int x = x0; x < x1; x += dx) {
            const int ix = gx(g[x]), iy = gy(g[x]);
            const int u = qa == 2 ? iy : ix, v = qa == 0 ? ix : iy;
            // the SIMD body multiplies floats, the tail converts the int product: both exact (|product| <= 4080^2 < 2^24)
            acc = __fadd_rn(acc, c < 4 ? __fmul_rn((float)u, (float)v) : (float)(u * v));
        }
    }
    return acc;
}

// One b chain: quantity qb (0: diff*Ix, 1: diff*Iy), chain c (0..3: pair sums of columns (x, x + 4), x = c + 8m < nsimd;
// 4: the tail, one product per column)
__device__ float run_b_chain(const WinSmem& sm, int win, int nsimd, int qb, int c)
{
    float acc = 0.f;
    for (int y = 0; y < win; y++) {
        const uint32_t* g = sm.grad + y * LKW_MAX;
        const int16_t* d = sm.diff + y * LKW_MAX;
        if (c < 4) {
            for (int x = c; x < nsimd; x += 8) {
                const int p0 = qb ? gy(g[x]) : gx(g[x]), p1 = qb ? gy(g[x + 4]) : gx(g[x + 4]);
                acc = __fadd_rn(acc, (float)(p0 * (int)d[x] + p1 * (int)d[x + 4]));
            }
        } else {
            for (int x = nsimd; x < win; x++)
                acc = __fadd_rn(acc, (float)((int)d[x] * (qb ? gy(g[x]) : gx(g[x]))));
        }
    }
    return acc;
}

} // namespace

template <bool SIZED>
__global__ void __launch_bounds__(LKW_WARPS_PER_CTA * 32, LKW_CTAS_PER_SM)
k_lk_win(const LkArgs args, const int win)
{
    __shared__ WinSmem smem[LKW_WARPS_PER_CTA];
    const int lane = threadIdx.x & 31;
    WinSmem& sm = smem[threadIdx.x >> 5];
    const bool col_lane = lane < win;               // lane x owns window column x
    const int nsimd = (win / 8) * 8;
    const float half_win = (win - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (1 << 20);
    const int max_level = args.nlevels - 1;
    const int items = args.n_units * args.per_unit;
    // runner lane L sums chain L % 5 of quantity L / 5 (A: lanes 0..14, b: lanes 0..9)
    const int rq = lane / 5, rc = lane - rq * 5;

    for (;;) {
        int item = 0;
        if (lane == 0) item = atomicAdd(args.queue, 1);
        item = __shfl_sync(FULL, item, 0);
        if (item >= items) break;
        const int unit = item / args.per_unit;
        const int f = item - unit * args.per_unit;
        const int npts = args.n_pts ? args.n_pts[unit] : args.cap;
        if (f >= npts) continue;

        const size_t pbase = (size_t)unit * args.cap + f;
        const UnitParams& par = args.par[unit];
        const int max_iters = par.max_iters;
        const double eps2 = par.eps2;
        const float min_eig = par.min_eig;
        float2 pt = args.pts_in[pbase];

        for (int call = 0; call < args.ncalls; call++) {
            const int img_prev = args.img_plane0 + unit * args.imgs_per_unit + args.img_prev[call];
            const int img_next = args.img_plane0 + unit * args.imgs_per_unit + args.img_next[call];
            float2 nxt = make_float2(0.f, 0.f);
            int status = 1;
            float errv = 0.f;
            for (int level = max_level; level >= 0; level--) {
                do {                            // one level-solve; `break` = the reference's `continue`
                    int lw = args.lw[level], lh = args.lh[level];
                    if (SIZED) { lw = __ldg(&args.geo[img_prev].w[level]); lh = __ldg(&args.geo[img_prev].h[level]); }
                    const int pitch = args.pitch[level];
                    const float sc = 1.f / (float)(1 << level);
                    float px = pt.x * sc, py = pt.y * sc;
                    if (level == max_level) { nxt.x = px; nxt.y = py; }
                    else { nxt.x = nxt.x * 2.f; nxt.y = nxt.y * 2.f; }
                    px -= half_win; py -= half_win;
                    const int ipx = __float2int_rd(px), ipy = __float2int_rd(py);
                    if (ipx < -win || ipx >= lw || ipy < -win || ipy >= lh) {
                        if (level == 0) { status = 0; errv = 0.f; }
                        break;
                    }
                    float a = px - (float)ipx, b = py - (float)ipy;
                    int w00, w01, w10, w11;
                    bilinear_weights(a, b, w00, w01, w10, w11);

                    // ---- patch extraction: lane x walks column x of the I and dI windows -----------------------
                    __syncwarp();               // the previous level-solve's runners are done with the patch
                    if (col_lane) {
                        const size_t o = (size_t)(ipy + VO_PAD) * pitch + (ipx + VO_PAD + lane);
                        const uint8_t* src = args.img_base[level] + args.plane[level] * img_prev + o;
                        const uint32_t* dsrc = args.der_base[level] + args.plane[level] * img_prev + o;
                        int i0 = __ldg(src), i1 = __ldg(src + 1);
                        uint32_t d0 = __ldg(dsrc), d1 = __ldg(dsrc + 1);
                        for (int y = 0; y < win; y++) {
                            src += pitch; dsrc += pitch;
                            const int i2 = __ldg(src), i3 = __ldg(src + 1);
                            const uint32_t d2 = __ldg(dsrc), d3 = __ldg(dsrc + 1);
                            const int iv = (i0 * w00 + i1 * w01 + i2 * w10 + i3 * w11 + (1 << (W_BITS - 6))) >> (W_BITS - 5);
                            const int ix = (gx(d0) * w00 + gx(d1) * w01 + gx(d2) * w10 + gx(d3) * w11 + (1 << (W_BITS - 1))) >> W_BITS;
                            const int iy = (gy(d0) * w00 + gy(d1) * w01 + gy(d2) * w10 + gy(d3) * w11 + (1 << (W_BITS - 1))) >> W_BITS;
                            sm.ival[y * LKW_MAX + lane] = (int16_t)iv;
                            sm.grad[y * LKW_MAX + lane] = ((uint32_t)ix & 0xffffu) | ((uint32_t)iy << 16);
                            i0 = i2; i1 = i3; d0 = d2; d1 = d3;
                        }
                    }
                    __syncwarp();
                    float A11, A12, A22;
                    {
                        float acc = 0.f;
                        if (lane < 15) acc = run_a_chain(sm, win, nsimd, rq, rc);
                        const float tot = combine_chains(acc);
                        A11 = __fmul_rn(__shfl_sync(FULL, tot, 0), FLT_SCALE);
                        A12 = __fmul_rn(__shfl_sync(FULL, tot, 5), FLT_SCALE);
                        A22 = __fmul_rn(__shfl_sync(FULL, tot, 10), FLT_SCALE);
                    }
                    float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
                    {
                        const float dd = __fsub_rn(A11, A22);
                        const float rad = __fadd_rn(__fmul_rn(dd, dd), __fmul_rn(__fmul_rn(4.f, A12), A12));
                        const float minEig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(rad)), (float)(2 * win * win));
                        if (minEig < min_eig || D < 1.1920928955078125e-07f) {
                            if (level == 0) status = 0;
                            break;
                        }
                    }
                    D = __fdiv_rn(1.f, D);

                    // ---- Newton iterations ---------------------------------------------------------------------
                    const uint8_t* const jplane = args.img_base[level] + args.plane[level] * img_next;
                    float npx = nxt.x - half_win, npy = nxt.y - half_win;
                    float pdx = 0.f, pdy = 0.f;
                    for (int j = 0; j < max_iters; j++) {
                        const int inx = __float2int_rd(npx), iny = __float2int_rd(npy);
                        if (inx < -win || inx >= lw || iny < -win || iny >= lh) {
                            if (level == 0) status = 0;
                            break;
                        }
                        a = npx - (float)inx; b = npy - (float)iny;
                        bilinear_weights(a, b, w00, w01, w10, w11);
                        __syncwarp();           // the previous iteration's runners are done with the residuals
                        if (col_lane) {
                            const uint8_t* src = jplane + (size_t)(iny + VO_PAD) * pitch + (inx + VO_PAD + lane);
                            int j0 = __ldg(src), j1 = __ldg(src + 1);
                            for (int y = 0; y < win; y++) {
                                src += pitch;
                                const int j2 = __ldg(src), j3 = __ldg(src + 1);
                                const int jv = (j0 * w00 + j1 * w01 + j2 * w10 + j3 * w11 + (1 << (W_BITS - 6))) >> (W_BITS - 5);
                                sm.diff[y * LKW_MAX + lane] = (int16_t)(jv - sm.ival[y * LKW_MAX + lane]);
                                j0 = j2; j1 = j3;
                            }
                        }
                        __syncwarp();
                        float acc = 0.f;
                        if (lane < 10) acc = run_b_chain(sm, win, nsimd, rq, rc);
                        const float tot = combine_chains(acc);
                        const float b1 = __fmul_rn(__shfl_sync(FULL, tot, 0), FLT_SCALE);
                        const float b2 = __fmul_rn(__shfl_sync(FULL, tot, 5), FLT_SCALE);
                        const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, b2), __fmul_rn(A22, b1)), D);
                        const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, b1), __fmul_rn(A11, b2)), D);
                        npx = __fadd_rn(npx, dx); npy = __fadd_rn(npy, dy);
                        nxt.x = __fadd_rn(npx, half_win); nxt.y = __fadd_rn(npy, half_win);
                        if ((double)dx * (double)dx + (double)dy * (double)dy <= eps2) break;
                        // std::abs(double(x)) < 0.01 for a float x  <=>  |x| <= 0.01f (0.01f is the largest float below 0.01)
                        if (j > 0 && fabsf(__fadd_rn(dx, pdx)) <= 0.01f && fabsf(__fadd_rn(dy, pdy)) <= 0.01f) {
                            nxt.x = __fsub_rn(nxt.x, __fmul_rn(dx, 0.5f));
                            nxt.y = __fsub_rn(nxt.y, __fmul_rn(dy, 0.5f));
                            break;
                        }
                        pdx = dx; pdy = dy;
                    }

                    // ---- level 0 epilogue: final bounds re-check (+ err when requested) -------------------------
                    if (level == 0 && status) {
                        const float fxp = __fsub_rn(nxt.x, half_win), fyp = __fsub_rn(nxt.y, half_win);
                        const int inx = __float2int_rd(fxp), iny = __float2int_rd(fyp);
                        if (inx < -win || inx >= lw || iny < -win || iny >= lh) {
                            status = 0;
                        } else if (args.err_out) {
                            a = fxp - (float)inx; b = fyp - (float)iny;
                            bilinear_weights(a, b, w00, w01, w10, w11);
                            int s = 0;
                            if (col_lane) {
                                const uint8_t* src = jplane + (size_t)(iny + VO_PAD) * pitch + (inx + VO_PAD + lane);
                                int j0 = __ldg(src), j1 = __ldg(src + 1);
                                for (int y = 0; y < win; y++) {
                                    src += pitch;
                                    const int j2 = __ldg(src), j3 = __ldg(src + 1);
                                    const int jv = (j0 * w00 + j1 * w01 + j2 * w10 + j3 * w11 + (1 << (W_BITS - 6))) >> (W_BITS - 5);
                                    s += abs(jv - sm.ival[y * LKW_MAX + lane]);
                                    j0 = j2; j1 = j3;
                                }
                            }
                            // errval += |diff| is a float sum of integers whose total stays below 2^24: exact in any order
                            s = __reduce_add_sync(FULL, s);
                            errv = __fdiv_rn((float)s, (float)(32 * win * win));
                        }
                    }
                } while (0); // level-solve
            }
            if (lane == 0) {                    // the call's outputs; the next call starts from them
                const size_t o = (size_t)call * args.call_stride + pbase;
                args.pts_out[o] = nxt;
                args.status_out[o] = (uint8_t)status;
                if (args.err_out) args.err_out[o] = errv;
            }
            pt = nxt;
        }
    } // work queue

    // the last warp to retire resets the queue for the next launch that uses it (every warp of the grid passes here once,
    // after its last fetch)
    if (lane == 0) {
        const int total_warps = gridDim.x * LKW_WARPS_PER_CTA;
        if (atomicAdd(args.queue + 1, 1) == total_warps - 1) {
            args.queue[1] = 0;
            __threadfence();
            args.queue[0] = 0;
        }
    }
}

cudaError_t vo_launch_lk_win(const LkArgs& args, int win, int sm_count, cudaStream_t stream)
{
    const long items = (long)args.n_units * args.per_unit;
    if (items <= 0) return cudaSuccess;
    if (win < VO_WIN_MIN || win > VO_WIN_MAX) return cudaErrorInvalidValue;
    const long resident = (long)(sm_count > 0 ? sm_count : 132) * LKW_CTAS_PER_SM;
    long ctas = (items + LKW_WARPS_PER_CTA - 1) / LKW_WARPS_PER_CTA;
    if (ctas > resident) ctas = resident;
    const int thr = LKW_WARPS_PER_CTA * 32;
    if (args.geo) k_lk_win<true><<<(int)ctas, thr, 0, stream>>>(args, win);
    else k_lk_win<false><<<(int)ctas, thr, 0, stream>>>(args, win);
    return cudaGetLastError();
}
