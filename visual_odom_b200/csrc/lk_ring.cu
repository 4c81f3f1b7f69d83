// lk_ring.cu -- K2: the pyramidal Lucas-Kanade kernel (the hot kernel of this library).
//
// Replaces the four chained cv::calcOpticalFlowPyrLK calls of the reference's circularMatching()
// (reference src/feature.cpp:136-139; window 21x21 :127, 30 iterations / eps 0.01 :128,
// maxLevel 3, minEigThreshold 1e-3 :136).  Arithmetic restated in oracle/lk_ref.c (lk_track),
// which is pinned bit-for-bit against cv2 4.13.0; this kernel reproduces the same bits:
//   * fixed-point bilinear patches (weights cvRound(w*2^14), DESCALE by 9 / 14)
//   * float32 normal equations accumulated in OpenCV's 4-SIMD-lane + scalar-tail order
//     (the order matters once partial sums pass 2^24; see "summation chains" below)
//   * per-level next = next*2 propagation, level-0-only status writes, final bounds re-check.
//
// Parallelisation: ONE WARP PER FEATURE-RING.  A feature's track never depends on another feature, so a warp
// runs the whole ring (up to 4 chained calls x all pyramid levels x <= 30 Newton iterations) of one feature
// and then takes the next feature from a global work queue (persistent warps: 8 CTAs of 2 warps per SM,
// every warp independent -- no CTA-level synchronisation after the start).  Ring durations differ by more
// than 2x between features (the iteration count is heavy-tailed), so static assignment would idle.
//
// Staging: per level, lane 0 issues three TMA (cp.async.bulk.tensor.3d) box loads into the warp's private
// shared memory: the 48x22 u8 window of the previous image, the 28x22 s16x2 window of its Scharr derivative,
// and a 48x32 u8 tile of the next image around the current estimate (re-issued only if the 22x22 search
// window drifts out of the tile).  The planes are physically padded (see common.cuh), so no box ever needs
// border handling.  The u8 windows are used where TMA writes them (row pitch 48 B): the work mapping below
// is chosen so that the rows a warp reads in one LDS fall into different banks at that pitch.
//
// Summation chains: OpenCV accumulates A11/A12/A22 and b1/b2 in float32 with 4 SIMD lanes over
// columns 0..15 (lane = x & 3) and a scalar tail over columns 16..20, rows outermost.  The 441
// window pixels are therefore split into 5 ordered chains (4 x 84 + 105 pixels); the addends of
// b are float(int pair sum) of columns (x, x+4).
//
// Work mapping (who computes which pixel): COLUMN STRIPS.  Lane L owns window column L>>1, rows
// 0..9 (L even) or 10..20 (L odd), plus 3 or 4 rows of one tail column (lanes 0..29).  A strip
// walks down its column, so the two byte taps of a row are fetched once (two aligned 32-bit loads
// + a funnel shift), serve as the bottom taps of one pixel and the top taps of the next, and feed
// the fixed-point bilinear interpolation as packed operands of dp2a.
//
// Summation (who adds): all addends are integers, so when the sum of |addend| over every chain is
// <= 2^24 each partial sum is exact and the chain totals are integer warp reductions (REDUX) --
// the fast path.  Otherwise the float addends are written to shared memory in chain order and one
// RUNNER lane per (quantity, chain) adds them strictly in order with 128-bit loads.  The A sums
// always take the faithful path (they pass 2^24 on any corner-like texture).
//
// Shared memory is re-used over a level's life: the derivative window is dead once the patch is extracted and then
// holds A22's chain slots; the packed I patch and the packed residuals stay in registers.  WarpSmem keeps the 8960 B
// layout that lets 24 warps fit per SM: shrinking it would move every shared-memory address, a change to be measured
// on its own.
#include "common.cuh"
#include "lk_ring.h"

#define FULL 0xffffffffu
#define W_BITS 14

namespace {

template <bool B> struct BoolC { static constexpr bool value = B; };

__device__ __forceinline__ uint32_t smem_u32(const void* p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2)
{
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
        "[%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ int ld_acquire(const int* p)
{
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int* p, int v)
{
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// generic-proxy accesses of a buffer (LDS/STS by this warp) before the async proxy (TMA) writes it again
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// per-warp shared memory
// TMA tile loads need a 16-byte aligned global start address, so every box starts at the
// 16-byte boundary at or below the wanted column and is 16 bytes wider than the data it must hold:
//   u8 windows  : 48 bytes wide  (<= 15 bytes of lead-in + 22 (I) / 32 (J) bytes of payload)
//   s16x2 window: 28 elements wide (<= 3 elements of lead-in + 22)
#define TW 48                   // row pitch (bytes) of the u8 windows = TMA box width.  12 words: rows d apart
                                // collide in the banks only for d = 8, 16; the strips of one LDS are 10 rows apart
                                // and the tail segments start at rows 0,3,7,10,14,17 (no two 8 or 16 apart)
#define TWW (TW / 4)
#define DW 28                   // row pitch (uint32) of the derivative box
#define I_ROWS 22
#define J_ROWS 32
// chain slots (floats): per quantity 4 SIMD slots of 84 + a tail slot of up to 116.  Slot starts in 16-byte
// units: 0,21,42,63,84 (+113 for the second quantity): all distinct mod 8 within each group of 8 runner
// lanes, so their 128-bit loads hit distinct bank groups.  A22's slots live in the dead derivative window,
// shifted by 2 units for the same reason.
#define SLOT_S 84
#define TAIL_OFF 336
#define QSTRIDE 452
#define A22_OFF 8               // words into dwin
struct __align__(128) WarpSmem {
    uint8_t jtile[TW * J_ROWS];             // next-image tile                                             1536
    uint8_t iwin[TW * I_ROWS + 96];         // previous-image window; afterwards the packed I patch       1152
    uint32_t dwin[DW * I_ROWS + 24];        // derivative window; then A22 chain slots; then residuals    2560
    float chain[2 * QSTRIDE];               // chain-ordered float addends of two quantities              3616
    uint64_t bar;                           // mbarrier for TMA completion
    uint64_t pad_[11];
};
static_assert(sizeof(WarpSmem) == 8960, "WarpSmem layout");
static_assert(A22_OFF + QSTRIDE <= DW * I_ROWS + 24, "A22 slots must fit the derivative window");

#define I_BYTES (TW * I_ROWS)
#define J_BYTES (TW * J_ROWS)
#define D_BYTES (DW * I_ROWS * 4)

// plain-load staging of one box (debug / A-B path): rows x 48 bytes from a padded plane
__device__ __forceinline__ void ldg_box_u8(uint8_t* dst, const uint8_t* plane, int pitch, int x, int y, int rows, int lane)
{
    const uint8_t* src = plane + (size_t)y * pitch + x;
    for (int r = 0; r < rows; r++) {
        dst[r * TW + lane] = __ldg(src + (size_t)r * pitch + lane);
        if (lane < TW - 32) dst[r * TW + 32 + lane] = __ldg(src + (size_t)r * pitch + 32 + lane);
    }
}
__device__ __forceinline__ void ldg_box_u32(uint32_t* dst, const uint32_t* plane, int pitch, int x, int y, int lane)
{
    const uint32_t* src = plane + (size_t)y * pitch + x;
    if (lane < DW)
        for (int r = 0; r < I_ROWS; r++) dst[r * DW + lane] = __ldg(src + (size_t)r * pitch + lane);
}

__device__ __forceinline__ void bilinear_weights(float a, float b, int& w00, int& w01, int& w10, int& w11)
{
    w00 = __float2int_rn((1.f - a) * (1.f - b) * (float)(1 << W_BITS));
    w01 = __float2int_rn(a * (1.f - b) * (float)(1 << W_BITS));
    w10 = __float2int_rn((1.f - a) * b * (float)(1 << W_BITS));
    w11 = (1 << W_BITS) - w00 - w01 - w10;
}

// a.lo * b.byte0 + a.hi * b.byte1 + c with SIGNED 16-bit halves of a (w11 = 2^14 - w00 - w01 - w10 can be -1)
// and UNSIGNED bytes of b: the two horizontal taps of the fixed-point bilinear interpolation
__device__ __forceinline__ int dp2a_taps(unsigned w_pair, unsigned taps, int c)
{
    int d;
    asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(w_pair), "r"(taps), "r"(c));
    return d;
}

// sum over the 8 lanes of a SIMD chain: lanes that differ only in bit 0 (row half) and bits 3,4
// (column group) -- every lane ends up with its own chain's total
__device__ __forceinline__ unsigned chain_sum_u(unsigned v)
{
    v += __shfl_xor_sync(FULL, v, 1);
    v += __shfl_xor_sync(FULL, v, 8);
    v += __shfl_xor_sync(FULL, v, 16);
    return v;
}

__device__ __forceinline__ float add4(float acc, const float4 t)
{
    acc = __fadd_rn(acc, t.x); acc = __fadd_rn(acc, t.y); acc = __fadd_rn(acc, t.z);
    return __fadd_rn(acc, t.w);
}
// Faithful float chains.  The addends of every chain lie contiguously, in chain order, in shared memory; one
// RUNNER lane per (quantity, chain) adds them strictly in order.  A SIMD chain has NS addends (84 for A, 42
// for b: pair sums), the tail chain 105.  Runner lanes execute this inside a divergent branch (the other lanes
// skip it), SIMD and tail runners share the first NS/4 vector steps.
template <int NS>
__device__ __forceinline__ float run_chain(const float* slot, bool is_tail)
{
    float acc = 0.f;
    const float4* p = reinterpret_cast<const float4*>(slot);
#pragma unroll
    for (int v = 0; v < NS / 4; v++) acc = add4(acc, p[v]);
    if (is_tail) {
#pragma unroll
        for (int v = NS / 4; v < 26; v++) acc = add4(acc, p[v]);
        acc = __fadd_rn(acc, slot[104]);
    } else if (NS % 4) {            // 42 = 10 vectors + 2
        const float2 t = *reinterpret_cast<const float2*>(slot + (NS / 4) * 4);
        acc = __fadd_rn(acc, t.x); acc = __fadd_rn(acc, t.y);
    }
    return acc;
}
// totals of the quantities held by the runner lanes 5q..5q+4:  tail + ((c0 + c2) + (c1 + c3)), formed in lane 5q
__device__ __forceinline__ float combine_chains(float acc)
{
    const float t1 = __fadd_rn(acc, __shfl_down_sync(FULL, acc, 2));     // lane 5q: c0 + c2, lane 5q+1: c1 + c3
    const float t2 = __fadd_rn(t1, __shfl_down_sync(FULL, t1, 1));       // lane 5q: (c0 + c2) + (c1 + c3)
    return __fadd_rn(__shfl_down_sync(FULL, acc, 4), t2);                // + tail
}

} // namespace

// ---------------------------------------------------------------------------------------------
// SIZED: the units' images have sizes of their own (args.geo); the other instantiation is the launch-wide-size kernel
// exactly, so runs of one image size pay nothing for the table
template <bool USE_TMA, bool SIZED>
__global__ void __launch_bounds__(LK_WARPS_PER_CTA * 32, LK_CTAS_PER_SM)
k_lk_ring(const __grid_constant__ LkMaps maps, const LkArgs args)
{
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int lane = threadIdx.x & 31;
    WarpSmem& sm = reinterpret_cast<WarpSmem*>(smem_raw)[threadIdx.x >> 5];

    // ---- static work mapping -------------------------------------------------------------------
    const int col = lane >> 1, half = lane & 1;
    const int r0 = half ? 10 : 0;                  // strip rows [r0, r0 + nvalid): 0..9 / 10..20
    const int nvalid_s = half ? 11 : 10;           // the 11th element of the even lanes is a dummy (zero gradient)
    const int chain = col & 3, cpos = col >> 2;    // SIMD chain and position inside the row's group of 4
    const bool has_tail = lane < 30;
    const int tcol = has_tail ? 16 + lane / 6 : 16;
    const int seg = lane % 6;
    // tail rows [tr0, tr0 + tn): segments of 3,4,3,4,3,4 rows starting at 0,3,7,10,14,17
    const int tr0 = has_tail ? (seg * 7) >> 1 : 0;
    const int tn = has_tail ? 3 + (seg & 1) : 0;
    // chain-buffer positions (floats) inside a quantity's slots.
    //   A (setup)     : SIMD element (row, col) at chain*84 + row*4 + cpos ; tail element at 336 + row*5 + (tcol-16)
    //   b (iteration) : SIMD pair (col, col+4) of a row at chain*84 + row*2 + cpos/2 (written by the even-cpos lane)
    const int a_pos = chain * SLOT_S + r0 * 4 + cpos;
    const int b_pos = chain * SLOT_S + r0 * 2 + (cpos >> 1);
    const int t_pos = TAIL_OFF + tr0 * 5 + (tcol - 16);
    // runner lane L sums slot (quantity L/5, chain L%5)
    const int rq = lane / 5, rc = lane - rq * 5;
    const int run_off = rc < 4 ? rc * SLOT_S : TAIL_OFF;
    const float* const run_slot = (rq < 2 ? sm.chain + rq * QSTRIDE : reinterpret_cast<const float*>(sm.dwin) + A22_OFF) + run_off;
    float* const a22 = reinterpret_cast<float*>(sm.dwin) + A22_OFF;

    if (USE_TMA) {
        if (lane == 0) {
            mbar_init(&sm.bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    uint32_t phase = 0;

    const float half_win = (VO_WIN - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (1 << 20);
    // delta.ddot(delta) <= eps^2 is a double test in OpenCV; dx*dx + dy*dy in float is within 2e-7 of it, so the double
    // form is only evaluated inside this band
    const float eps2_lo = (float)(args.eps2 * 0.999999), eps2_hi = (float)(args.eps2 * 1.000001);
    const int max_level = args.nlevels - 1;
    // Work items.  A feature-ring is ncalls x nlevels PHASES (one level-solve each).  An item is `span`
    // consecutive phases of one feature; items are queued phase-major, so every feature's phase p is handed out
    // before any feature's phase p + span.  span = all phases gives one item per feature-ring (no hand-over);
    // a small span bounds the tail of a launch by one level-solve instead of one whole ring (the ring cost is
    // heavy-tailed: max / mean = 3.4).  The state handed from item to item is the running estimate (pts_out)
    // and a per-feature progress counter; an item waits for its predecessor, which was dequeued earlier by a
    // running warp, so the wait always ends.
    const int nphases = args.ncalls * args.nlevels;
    const int span = args.span > 0 && args.span < nphases ? args.span : nphases;
    const int per_group = args.n_units * args.per_unit;
    const int items = ((nphases + span - 1) / span) * per_group;

    for (;;) {
        int item = 0;
        if (lane == 0) item = atomicAdd(args.queue, 1);
        item = __shfl_sync(FULL, item, 0);
        if (item >= items) break;
        const int grp = item / per_group;
        const int rem = item - grp * per_group;
        const int unit = rem / args.per_unit;
        const int f = rem - unit * args.per_unit;
        const int npts = args.n_pts ? args.n_pts[unit] : args.cap;
        if (f >= npts) continue;

        const size_t pbase = (size_t)unit * args.cap + f;
        const int p0 = grp * span, p1 = min(p0 + span, nphases);
        if (p0 > 0) {                           // the predecessor item has published its state
            if (lane == 0)
                while (ld_acquire(args.progress + pbase) < p0) __nanosleep(64);
            __syncwarp();
        }
        int call = p0 / args.nlevels;
        float2 pt = call == 0 ? args.pts_in[pbase] : __ldcg(args.pts_out + (size_t)(call - 1) * args.call_stride + pbase);
        float2 nxt = make_float2(0.f, 0.f);
        if (p0 - call * args.nlevels > 0) nxt = __ldcg(args.pts_out + (size_t)call * args.call_stride + pbase);
        int status = 1;
        float errv = 0.f;

        for (int ph = p0; ph < p1; ph++) {
            call = ph / args.nlevels;
            const int level = max_level - (ph - call * args.nlevels);
            const int img_prev = args.img_plane0 + unit * args.imgs_per_unit + args.img_prev[call];
            const int img_next = args.img_plane0 + unit * args.imgs_per_unit + args.img_next[call];
            do {                                // one level-solve; `break` = the reference's `continue`
                int lw = args.lw[level], lh = args.lh[level];
                if (SIZED) { lw = __ldg(&args.geo[img_prev].w[level]); lh = __ldg(&args.geo[img_prev].h[level]); }
                const float sc = 1.f / (float)(1 << level);
                float px = pt.x * sc, py = pt.y * sc;
                if (level == max_level) { nxt.x = px; nxt.y = py; }
                else { nxt.x = nxt.x * 2.f; nxt.y = nxt.y * 2.f; }
                px -= half_win; py -= half_win;
                const int ipx = __float2int_rd(px), ipy = __float2int_rd(py);
                if (ipx < -VO_WIN || ipx >= lw || ipy < -VO_WIN || ipy >= lh) {
                    if (level == 0) { status = 0; errv = 0.f; }
                    break;
                }
                // ---- stage windows: I (u8), dI (s16x2), J tile (u8) --------------------------------
                float npx = nxt.x - half_win, npy = nxt.y - half_win;
                int inx = __float2int_rd(npx), iny = __float2int_rd(npy);
                const bool j_ok0 = !(inx < -VO_WIN || inx >= lw || iny < -VO_WIN || iny >= lh);
                // box origins in padded-plane coordinates, x snapped down to the 16-byte boundary
                const int ibx = (ipx + VO_PAD) & ~15, iby = ipy + VO_PAD;       // u8 window of I
                const int dbx = (ipx + VO_PAD) & ~3;                            // derivative window (4 elements = 16 B)
                int jbx = (inx - 5 + VO_PAD) & ~15, jby = iny - 5 + VO_PAD;     // tile of J
                __syncwarp();
                if (USE_TMA) {
                    if (lane == 0) {
                        fence_proxy_async();
                        mbar_expect_tx(&sm.bar, I_BYTES + D_BYTES + (j_ok0 ? J_BYTES : 0));
                        tma_load_3d(sm.iwin, &maps.img_i[level], &sm.bar, ibx, iby, img_prev);
                        tma_load_3d(sm.dwin, &maps.der[level], &sm.bar, dbx, iby, img_prev);
                        if (j_ok0)
                            tma_load_3d(sm.jtile, &maps.img_j[level], &sm.bar, jbx, jby, img_next);
                    }
                } else {
                    ldg_box_u8(sm.iwin, args.img_base[level] + args.plane[level] * img_prev, args.pitch[level], ibx, iby, I_ROWS, lane);
                    ldg_box_u32(sm.dwin, args.der_base[level] + args.plane[level] * img_prev, args.pitch[level], dbx, iby, lane);
                    if (j_ok0)
                        ldg_box_u8(sm.jtile, args.img_base[level] + args.plane[level] * img_next, args.pitch[level], jbx, jby, J_ROWS, lane);
                    __syncwarp();
                }
                float a = px - (float)ipx, b = py - (float)ipy;
                int w00, w01, w10, w11;
                bilinear_weights(a, b, w00, w01, w10, w11);
                if (USE_TMA) { mbar_wait(&sm.bar, phase); phase ^= 1; }

                // ---- patch extraction: I (x32), Ix, Iy of the strip elements; A addends in chain order ----
                int dxy[15];          // lo16 = Ix, hi16 = Iy
                int Ipk[8];           // int16 patch intensities, two per register: strip 0..10, tail 11..14
                float A11, A12, A22;
                {
                    float a22v[15];       // A22 addends: their slots alias the derivative window, stored after the extraction
                    const unsigned wt = (unsigned)w00 | ((unsigned)w01 << 16), wb = (unsigned)w10 | ((unsigned)(w11 & 0xffff) << 16);
                    const int ox = ipx + VO_PAD - ibx, odx = ipx + VO_PAD - dbx;
#pragma unroll
                    for (int part = 0; part < 2; part++) {
                        const int c0 = part ? tcol : col, row0 = part ? tr0 : r0, ne = part ? 4 : 11, nvalid = part ? tn : nvalid_s;
                        const int ioff = row0 * TW + ox + c0;                      // byte offset of the strip's first tap
                        const uint32_t* iw = reinterpret_cast<const uint32_t*>(sm.iwin) + (ioff >> 2);
                        const int ish = 8 * (ioff & 3);
                        const uint32_t* dw = sm.dwin + row0 * DW + odx + c0;
                        unsigned ptop = __funnelshift_r(iw[0], iw[1], ish);
                        unsigned d00 = dw[0], d01 = dw[1];
#pragma unroll
                        for (int k = 0; k < ne; k++) {
                            // a dummy element (k >= nvalid) reads rows that exist (<= row 21 of the windows) and is zeroed
                            const unsigned pbot = __funnelshift_r(iw[(k + 1) * TWW], iw[(k + 1) * TWW + 1], ish);
                            const unsigned d10 = dw[(k + 1) * DW], d11 = dw[(k + 1) * DW + 1];
                            const int ival = (dp2a_taps(wb, pbot, dp2a_taps(wt, ptop, 1 << (W_BITS - 6))) >> (W_BITS - 5));
                            int ix = ((int)(short)(d00 & 0xffff) * w00 + (int)(short)(d01 & 0xffff) * w01 +
                                      (int)(short)(d10 & 0xffff) * w10 + (int)(short)(d11 & 0xffff) * w11 + (1 << (W_BITS - 1))) >> W_BITS;
                            int iy = (((int)d00 >> 16) * w00 + ((int)d01 >> 16) * w01 +
                                      ((int)d10 >> 16) * w10 + ((int)d11 >> 16) * w11 + (1 << (W_BITS - 1))) >> W_BITS;
                            if (k >= nvalid) { ix = 0; iy = 0; }
                            const int e = part ? 11 + k : k;
                            if (e & 1) Ipk[e >> 1] |= ival << 16; else Ipk[e >> 1] = ival & 0xffff;
                            dxy[e] = (ix & 0xffff) | (iy << 16);
                            const float fx = (float)ix, fy = (float)iy;
                            const int pos = part ? t_pos + k * 5 : a_pos + k * 4;
                            // a dummy element's position belongs to another lane: no store
                            if (k < nvalid) {
                                sm.chain[pos] = __fmul_rn(fx, fx);
                                sm.chain[QSTRIDE + pos] = __fmul_rn(fx, fy);
                            }
                            a22v[e] = __fmul_rn(fy, fy);
                            ptop = pbot; d00 = d10; d01 = d11;
                        }
                    }
                    __syncwarp();                   // every lane has read its I / dI windows
#pragma unroll
                    for (int e = 0; e < 15; e++) {
                        const int k = e < 11 ? e : e - 11;
                        if (k < (e < 11 ? nvalid_s : tn)) a22[(e < 11 ? a_pos + k * 4 : t_pos + k * 5)] = a22v[e];
                    }
                    __syncwarp();
                    float acc = 0.f;
                    if (lane < 15) acc = run_chain<84>(run_slot, rc == 4);
                    const float tot = combine_chains(acc);
                    const float iA11 = __shfl_sync(FULL, tot, 0), iA12 = __shfl_sync(FULL, tot, 5), iA22 = __shfl_sync(FULL, tot, 10);
                    A11 = __fmul_rn(iA11, FLT_SCALE); A12 = __fmul_rn(iA12, FLT_SCALE); A22 = __fmul_rn(iA22, FLT_SCALE);
                    __syncwarp();
                }
                float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
                {
                    float dd = __fsub_rn(A11, A22);
                    float rad = __fadd_rn(__fmul_rn(dd, dd), __fmul_rn(__fmul_rn(4.f, A12), A12));
                    float minEig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(rad)), (float)(2 * VO_WIN * VO_WIN));
                    if (minEig < args.min_eig || D < 1.1920928955078125e-07f) {
                        if (level == 0) status = 0;
                        break;
                    }
                }
                D = __fdiv_rn(1.f, D);

                // ---- Newton iterations ------------------------------------------------------------
                float pdx = 0.f, pdy = 0.f;
                bool tile_valid = j_ok0;
                bool force_replay = false;          // set by the first faithful replay of this level-solve
                for (int j = 0; j < args.max_iters; j++) {
                    inx = __float2int_rd(npx); iny = __float2int_rd(npy);
                    if (inx < -VO_WIN || inx >= lw || iny < -VO_WIN || iny >= lh) {
                        if (level == 0) status = 0;
                        break;
                    }
                    int rx = inx + VO_PAD - jbx, ry = iny + VO_PAD - jby;   // window origin inside the tile
                    if (!tile_valid || rx < 0 || ry < 0 || rx > TW - 22 || ry > J_ROWS - 22) {
                        jbx = (inx - 5 + VO_PAD) & ~15; jby = iny - 5 + VO_PAD;
                        rx = inx + VO_PAD - jbx; ry = 5;
                        __syncwarp();
                        if (USE_TMA) {
                            if (lane == 0) {
                                fence_proxy_async();
                                mbar_expect_tx(&sm.bar, J_BYTES);
                                tma_load_3d(sm.jtile, &maps.img_j[level], &sm.bar, jbx, jby, img_next);
                            }
                            mbar_wait(&sm.bar, phase); phase ^= 1;
                        } else {
                            ldg_box_u8(sm.jtile, args.img_base[level] + args.plane[level] * img_next, args.pitch[level], jbx, jby, J_ROWS, lane);
                            __syncwarp();
                        }
                        tile_valid = true;
                    }
                    a = npx - (float)inx; b = npy - (float)iny;
                    bilinear_weights(a, b, w00, w01, w10, w11);
                    const unsigned wt = (unsigned)w00 | ((unsigned)w01 << 16), wb = (unsigned)w10 | ((unsigned)(w11 & 0xffff) << 16);
                    int sxs = 0, sys = 0, sxt = 0, syt = 0;         // signed sums: strip (my SIMD chain) / tail
                    unsigned axs = 0, ays = 0, axt = 0, ayt = 0;    // sums of |addend|
                    int dpk[8];                       // int16 residuals, two per register (same element order as the I patch)
                    // The residual pass.  WITH_SUMS: also the products with the gradients, their exact integer sums and the
                    // sums of |addend| that decide whether the integer sums ARE the float32 chain sums.  Once an iteration of
                    // a level needed the faithful replay the following ones nearly always do (oracle: 94 %), and the replay
                    // recomputes the products from the residuals anyway -- so after a replay the rest of the level runs the
                    // light pass and goes straight to the replay (always valid, only slower than the exact path).
                    auto residual_pass = [&](auto with_sums) {
                        constexpr bool WITH_SUMS = decltype(with_sums)::value;
#pragma unroll
                        for (int part = 0; part < 2; part++) {
                            const int c0 = part ? tcol : col, row0 = part ? tr0 : r0, ne = part ? 4 : 11;
                            const int joff = (ry + row0) * TW + rx + c0;
                            const uint32_t* jw = reinterpret_cast<const uint32_t*>(sm.jtile) + (joff >> 2);
                            const int jsh = 8 * (joff & 3);
                            unsigned ptop = __funnelshift_r(jw[0], jw[1], jsh);
#pragma unroll
                            for (int k = 0; k < ne; k++) {
                                const unsigned pbot = __funnelshift_r(jw[(k + 1) * TWW], jw[(k + 1) * TWW + 1], jsh);
                                const int e = part ? 11 + k : k;
                                const int Iv = (e & 1) ? (Ipk[e >> 1] >> 16) : (int)(short)(Ipk[e >> 1] & 0xffff);
                                const int diff = (dp2a_taps(wb, pbot, dp2a_taps(wt, ptop, 1 << (W_BITS - 6))) >> (W_BITS - 5)) - Iv;
                                if (e & 1) dpk[e >> 1] |= diff << 16; else dpk[e >> 1] = diff & 0xffff;
                                if (WITH_SUMS) {
                                    const int vx = diff * (int)(short)(dxy[e] & 0xffff);      // gradients are 0 for dummy elements
                                    const int vy = diff * (dxy[e] >> 16);
                                    // |v| + acc in one VABSDIFF (|v| <= 2^28, 15 of them per lane: no overflow)
                                    if (part) { sxt += vx; syt += vy; axt = __sad(vx, 0, axt); ayt = __sad(vy, 0, ayt); }
                                    else { sxs += vx; sys += vy; axs = __sad(vx, 0, axs); ays = __sad(vy, 0, ays); }
                                }
                                ptop = pbot;
                            }
                        }
                    };
                    bool exact = false;
                    if (force_replay) {
                        residual_pass(BoolC<false>{});
                    } else {
                        residual_pass(BoolC<true>{});
                        // per-chain totals (exact integers) and per-chain sums of |addend| (REDUX over the chain's lanes)
                        const unsigned cax = chain_sum_u(axs), cay = chain_sum_u(ays);
                        const unsigned tax = __reduce_add_sync(FULL, axt), tay = __reduce_add_sync(FULL, ayt);
                        // |pair sum| <= |v0| + |v1|, so the bound is conservative for the SIMD chains
                        exact = __all_sync(FULL, cax <= (1u << 24) && cay <= (1u << 24) && tax <= (1u << 24) && tay <= (1u << 24));
                    }
                    float ib1, ib2;
                    if (exact) {
                        // every partial sum of every chain is an exactly representable integer.
                        // chain c's total sits in lanes 2c (x) / 2c+1 (y): even lanes carry b1, odd lanes b2
                        const float fx = (float)(int)chain_sum_u((unsigned)sxs), fy = (float)(int)chain_sum_u((unsigned)sys);
                        const float tx = (float)__reduce_add_sync(FULL, sxt), ty = (float)__reduce_add_sync(FULL, syt);
                        const float v = half ? fy : fx;
                        const float t1 = __fadd_rn(v, __shfl_down_sync(FULL, v, 4));      // lanes 0/1: c0 + c2, lanes 2/3: c1 + c3
                        const float t2 = __fadd_rn(t1, __shfl_down_sync(FULL, t1, 2));    // lanes 0/1: (c0 + c2) + (c1 + c3)
                        const float tot = __fadd_rn(half ? ty : tx, t2);
                        ib1 = __shfl_sync(FULL, tot, 0); ib2 = __shfl_sync(FULL, tot, 1);
                    } else {
                        // faithful replay: float addends in chain order, runner lanes add them
#pragma unroll
                        for (int k = 0; k < 11; k++) {
                            const int d = (k & 1) ? (dpk[k >> 1] >> 16) : (int)(short)(dpk[k >> 1] & 0xffff);
                            const int vx = d * (int)(short)(dxy[k] & 0xffff), vy = d * (dxy[k] >> 16);
                            const int px2 = vx + __shfl_down_sync(FULL, vx, 8), py2 = vy + __shfl_down_sync(FULL, vy, 8);   // + column x+4
                            if (!(cpos & 1) && k < nvalid_s) {
                                sm.chain[b_pos + k * 2] = (float)px2;
                                sm.chain[QSTRIDE + b_pos + k * 2] = (float)py2;
                            }
                        }
#pragma unroll
                        for (int k = 0; k < 4; k++) {
                            const int e = 11 + k;
                            const int d = (e & 1) ? (dpk[e >> 1] >> 16) : (int)(short)(dpk[e >> 1] & 0xffff);
                            if (k < tn) {
                                sm.chain[t_pos + k * 5] = (float)(d * (int)(short)(dxy[e] & 0xffff));
                                sm.chain[QSTRIDE + t_pos + k * 5] = (float)(d * (dxy[e] >> 16));
                            }
                        }
                        __syncwarp();
                        float acc = 0.f;
                        force_replay = true;
                        if (lane < 10) acc = run_chain<42>(run_slot, rc == 4);
                        const float tot = combine_chains(acc);
                        ib1 = __shfl_sync(FULL, tot, 0); ib2 = __shfl_sync(FULL, tot, 5);
                        __syncwarp();
                    }
                    const float b1 = __fmul_rn(ib1, FLT_SCALE), b2 = __fmul_rn(ib2, FLT_SCALE);
                    const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, b2), __fmul_rn(A22, b1)), D);
                    const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, b1), __fmul_rn(A11, b2)), D);
                    npx = __fadd_rn(npx, dx); npy = __fadd_rn(npy, dy);
                    nxt.x = __fadd_rn(npx, half_win); nxt.y = __fadd_rn(npy, half_win);
                    {
                        const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
                        if (d2 < eps2_lo) break;
                        if (d2 <= eps2_hi && (double)dx * (double)dx + (double)dy * (double)dy <= args.eps2) break;
                    }
                    // std::abs(double(x)) < 0.01 for a float x  <=>  |x| <= 0.01f (0.01f is the largest float below 0.01)
                    if (j > 0 && fabsf(__fadd_rn(dx, pdx)) <= 0.01f && fabsf(__fadd_rn(dy, pdy)) <= 0.01f) {
                        nxt.x = __fsub_rn(nxt.x, __fmul_rn(dx, 0.5f));
                        nxt.y = __fsub_rn(nxt.y, __fmul_rn(dy, 0.5f));
                        break;
                    }
                    pdx = dx; pdy = dy;
                }

                // ---- level 0 epilogue: final bounds re-check (+ err when requested) ---------------
                if (level == 0 && status) {
                    float fxp = __fsub_rn(nxt.x, half_win), fyp = __fsub_rn(nxt.y, half_win);
                    inx = __float2int_rd(fxp); iny = __float2int_rd(fyp);
                    if (inx < -VO_WIN || inx >= lw || iny < -VO_WIN || iny >= lh) {
                        status = 0;
                    } else if (args.err_out) {
                        int rx = inx + VO_PAD - jbx, ry = iny + VO_PAD - jby;
                        if (!tile_valid || rx < 0 || ry < 0 || rx > TW - 22 || ry > J_ROWS - 22) {
                            jbx = (inx - 5 + VO_PAD) & ~15; jby = iny - 5 + VO_PAD;
                            rx = inx + VO_PAD - jbx; ry = 5;
                            __syncwarp();
                            if (USE_TMA) {
                                if (lane == 0) {
                                    fence_proxy_async();
                                    mbar_expect_tx(&sm.bar, J_BYTES);
                                    tma_load_3d(sm.jtile, &maps.img_j[0], &sm.bar, jbx, jby, img_next);
                                }
                                mbar_wait(&sm.bar, phase); phase ^= 1;
                            } else {
                                ldg_box_u8(sm.jtile, args.img_base[0] + args.plane[0] * img_next, args.pitch[0], jbx, jby, J_ROWS, lane);
                                __syncwarp();
                            }
                        }
                        a = fxp - (float)inx; b = fyp - (float)iny;
                        bilinear_weights(a, b, w00, w01, w10, w11);
                        const unsigned wt = (unsigned)w00 | ((unsigned)w01 << 16), wb = (unsigned)w10 | ((unsigned)(w11 & 0xffff) << 16);
                        // errval += |diff| is a plain row-major float sum of small integers
                        // (<= 441 * 8160 < 2^24): exact, so any order gives the same float.
                        int s = 0;
#pragma unroll
                        for (int part = 0; part < 2; part++) {
                            const int c0 = part ? tcol : col, row0 = part ? tr0 : r0, ne = part ? 4 : 11, nvalid = part ? tn : nvalid_s;
                            const int joff = (ry + row0) * TW + rx + c0;
                            const uint32_t* jw = reinterpret_cast<const uint32_t*>(sm.jtile) + (joff >> 2);
                            const int jsh = 8 * (joff & 3);
                            unsigned ptop = __funnelshift_r(jw[0], jw[1], jsh);
#pragma unroll
                            for (int k = 0; k < ne; k++) {
                                const unsigned pbot = __funnelshift_r(jw[(k + 1) * TWW], jw[(k + 1) * TWW + 1], jsh);
                                const int e = part ? 11 + k : k;
                                const int Iv = (e & 1) ? (Ipk[e >> 1] >> 16) : (int)(short)(Ipk[e >> 1] & 0xffff);
                                const int diff = (dp2a_taps(wb, pbot, dp2a_taps(wt, ptop, 1 << (W_BITS - 6))) >> (W_BITS - 5)) - Iv;
                                if (k < nvalid) s += abs(diff);
                                ptop = pbot;
                            }
                        }
                        s = __reduce_add_sync(FULL, s);
                        errv = __fdiv_rn(__fmul_rn((float)s, 1.f), (float)(32 * VO_WIN * VO_WIN));
                    }
                }
            } while (0); // level-solve

            if (level == 0) {                   // end of a call: its outputs; the next call starts from them
                if (lane == 0) {
                    const size_t o = (size_t)call * args.call_stride + pbase;
                    args.pts_out[o] = nxt;
                    args.status_out[o] = (uint8_t)status;
                    if (args.err_out) args.err_out[o] = errv;
                }
                pt = nxt;
                status = 1; errv = 0.f;
            }
        } // phases of this item
        if (span < nphases && lane == 0) {
            const int last_level = max_level - ((p1 - 1) - call * args.nlevels);
            if (last_level != 0) args.pts_out[(size_t)call * args.call_stride + pbase] = nxt;    // running estimate
            st_release(args.progress + pbase, p1 == nphases ? 0 : p1);     // the last item leaves the counter clean
        }
    } // work queue

    // the last warp to retire resets the queue for the next launch that uses it (every warp of the grid passes here once,
    // after its last fetch)
    if (lane == 0) {
        const int total_warps = gridDim.x * LK_WARPS_PER_CTA;
        if (atomicAdd(args.queue + 1, 1) == total_warps - 1) {
            args.queue[1] = 0;
            __threadfence();
            args.queue[0] = 0;
        }
    }
}

// ---------------------------------------------------------------------------------------------
size_t vo_lk_smem_bytes() { return sizeof(WarpSmem) * LK_WARPS_PER_CTA; }

template <bool T, bool S>
static cudaError_t prep()
{
    return cudaFuncSetAttribute(k_lk_ring<T, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vo_lk_smem_bytes());
}

cudaError_t vo_lk_prepare()
{
    cudaError_t e = prep<false, false>();
    if (e == cudaSuccess) e = prep<true, false>();
    if (e == cudaSuccess) e = prep<false, true>();
    return e != cudaSuccess ? e : prep<true, true>();
}

cudaError_t vo_launch_lk_ring(const LkMaps& maps, const LkArgs& args, int sm_count, cudaStream_t stream)
{
    const long items = (long)args.n_units * args.per_unit;          // features; every feature has (nphases / span) work items
    if (items <= 0) return cudaSuccess;
    const long resident = (long)(sm_count > 0 ? sm_count : 148) * LK_CTAS_PER_SM;
    long ctas = (items + LK_WARPS_PER_CTA - 1) / LK_WARPS_PER_CTA;
    if (ctas > resident) ctas = resident;
    const int thr = LK_WARPS_PER_CTA * 32;
    const size_t sh = vo_lk_smem_bytes();
    if (args.geo) {
        if (args.use_tma) k_lk_ring<true, true><<<(int)ctas, thr, sh, stream>>>(maps, args);
        else k_lk_ring<false, true><<<(int)ctas, thr, sh, stream>>>(maps, args);
    } else if (args.use_tma) k_lk_ring<true, false><<<(int)ctas, thr, sh, stream>>>(maps, args);
    else k_lk_ring<false, false><<<(int)ctas, thr, sh, stream>>>(maps, args);
    return cudaGetLastError();
}
