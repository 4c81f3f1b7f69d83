/*
 * oracle/lk_ref.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * Plain-C CPU restatement of the arithmetic behind the reference's
 *   cv::calcOpticalFlowPyrLK(prev, next, prevPts, nextPts, status, err,
 *                            Size(21,21), 3, TermCriteria(COUNT+EPS,30,0.01), 0, 0.001)
 * call sites (reference src/feature.cpp:136-139, src/feature.cpp:72).  The
 * arithmetic itself lives in OpenCV (un-vendored third-party dependency; this
 * build is pinned to OpenCV 4.13.0 as installed, modules/video/src/lkpyramid.cpp,
 * modules/imgproc/src/pyramids.cpp -- sources are not on disk, the published
 * algorithm is restated here and pinned bit-for-bit against cv2 4.13.0 by
 * tests/test_oracle_lk.py).
 *
 * Restated pieces (SURVEY.md section 8a row A2):
 *   pyr_down_u8        5x5 [1 4 6 4 1]^2 REFLECT_101, (s+128)>>8, dst=((w+1)/2,(h+1)/2)
 *   scharr_deriv       int16x2 interleaved Scharr derivative, REFLECT_101
 *   lk_track           per-point coarse-to-fine LK with fixed-point patches,
 *                      float32 normal equations, OpenCV's SIMD-lane float
 *                      summation order (so the result is bit-identical, not
 *                      merely close), status / err semantics.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>

static inline int reflect101(int p, int len)
{
    if (len == 1) return 0;
    while (p < 0 || p >= len) {
        if (p < 0) p = -p;
        else p = 2 * len - 2 - p;
    }
    return p;
}

/* cv::pyrDown for CV_8UC1, BORDER_REFLECT_101 (default). */
void pyr_down_u8(const uint8_t *src, int w, int h, int sstep,
                 uint8_t *dst, int dstep)
{
    int dw = (w + 1) / 2, dh = (h + 1) / 2;
    static const int k[5] = {1, 4, 6, 4, 1};
    for (int y = 0; y < dh; y++) {
        for (int x = 0; x < dw; x++) {
            int s = 0;
            for (int j = 0; j < 5; j++) {
                int sy = reflect101(2 * y + j - 2, h);
                int r = 0;
                for (int i = 0; i < 5; i++) {
                    int sx = reflect101(2 * x + i - 2, w);
                    r += k[i] * src[sy * sstep + sx];
                }
                s += k[j] * r;
            }
            dst[y * dstep + x] = (uint8_t)((s + 128) >> 8);
        }
    }
}

/* calcScharrDeriv: d[2*x] = dI/dx, d[2*x+1] = dI/dy (int16), REFLECT_101. */
void scharr_deriv(const uint8_t *src, int w, int h, int sstep,
                  int16_t *dst, int dstep /* in int16 elements */)
{
    for (int y = 0; y < h; y++) {
        const uint8_t *r0 = src + reflect101(y - 1, h) * sstep;
        const uint8_t *r1 = src + y * sstep;
        const uint8_t *r2 = src + reflect101(y + 1, h) * sstep;
        for (int x = 0; x < w; x++) {
            int xm = reflect101(x - 1, w), xp = reflect101(x + 1, w);
            int t0m = (r0[xm] + r2[xm]) * 3 + r1[xm] * 10;
            int t0p = (r0[xp] + r2[xp]) * 3 + r1[xp] * 10;
            int t1m = r2[xm] - r0[xm];
            int t1c = r2[x] - r0[x];
            int t1p = r2[xp] - r0[xp];
            dst[y * dstep + 2 * x] = (int16_t)(t0p - t0m);
            dst[y * dstep + 2 * x + 1] = (int16_t)((t1m + t1p) * 3 + t1c * 10);
        }
    }
}

/* ------------------------------------------------------------------------- */

typedef struct {
    int w, h;           /* image size of this level              */
    int pad;            /* border of the padded copies            */
    int istep;          /* row stride of padded u8 image          */
    uint8_t *img;       /* padded REFLECT_101 image, origin at (pad,pad) */
    int dstep;          /* row stride (int16 elements) of padded derivative */
    int16_t *deriv;     /* zero-padded Scharr derivative (interleaved) or NULL */
} lk_level_t;

typedef struct {
    int nlevels;        /* number of pyramid images (= effective maxLevel+1) */
    lk_level_t lv[16];
} lk_pyr_t;

static void pad_reflect101(const uint8_t *src, int w, int h, int sstep,
                           uint8_t *dst, int pad, int dstep)
{
    for (int y = -pad; y < h + pad; y++) {
        int sy = reflect101(y, h);
        for (int x = -pad; x < w + pad; x++) {
            int sx = reflect101(x, w);
            dst[(y + pad) * dstep + (x + pad)] = src[sy * sstep + sx];
        }
    }
}

/* buildOpticalFlowPyramid(img, pyr, winSize, maxLevel, withDerivatives, REFLECT_101, CONSTANT) */
lk_pyr_t *lk_pyr_build(const uint8_t *img, int w, int h, int step,
                       int win, int max_level, int with_deriv)
{
    lk_pyr_t *p = (lk_pyr_t *)calloc(1, sizeof(lk_pyr_t));
    int pad = win;
    const uint8_t *cur = img;
    int cw = w, ch = h, cstep = step;
    uint8_t *tmp_prev = NULL;
    for (int l = 0; l <= max_level; l++) {
        uint8_t *tmp = NULL;
        if (l > 0) {
            int nw = (cw + 1) / 2, nh = (ch + 1) / 2;
            /* OpenCV stops when the level is not larger than the window */
            if (nw <= win || nh <= win) break;
            tmp = (uint8_t *)malloc((size_t)nw * nh);
            pyr_down_u8(cur, cw, ch, cstep, tmp, nw);
            cur = tmp; cw = nw; ch = nh; cstep = nw;
        }
        lk_level_t *L = &p->lv[l];
        L->w = cw; L->h = ch; L->pad = pad;
        L->istep = cw + 2 * pad;
        L->img = (uint8_t *)malloc((size_t)L->istep * (ch + 2 * pad));
        pad_reflect101(cur, cw, ch, cstep, L->img, pad, L->istep);
        if (with_deriv) {
            L->dstep = 2 * (cw + 2 * pad);
            L->deriv = (int16_t *)calloc((size_t)L->dstep * (ch + 2 * pad), sizeof(int16_t));
            scharr_deriv(cur, cw, ch, cstep,
                         L->deriv + pad * L->dstep + 2 * pad, L->dstep);
        }
        p->nlevels = l + 1;
        if (tmp_prev) free(tmp_prev);
        tmp_prev = tmp;
    }
    if (tmp_prev) free(tmp_prev);
    return p;
}

void lk_pyr_free(lk_pyr_t *p)
{
    if (!p) return;
    for (int l = 0; l < p->nlevels; l++) { free(p->lv[l].img); free(p->lv[l].deriv); }
    free(p);
}

int lk_pyr_nlevels(const lk_pyr_t *p) { return p->nlevels; }
void lk_pyr_level_info(const lk_pyr_t *p, int l, int *w, int *h, int *pad, int *istep)
{ *w = p->lv[l].w; *h = p->lv[l].h; *pad = p->lv[l].pad; *istep = p->lv[l].istep; }
const uint8_t *lk_pyr_level_img(const lk_pyr_t *p, int l) { return p->lv[l].img; }
const int16_t *lk_pyr_level_deriv(const lk_pyr_t *p, int l) { return p->lv[l].deriv; }

/* ------------------------------------------------------------------------- */
/* accumulation-order selector (the pinned one is mode 0; the others exist so
 * tests can show that the order matters and that mode 0 is the cv2 one).  oracle/cref.py names them (SUM_*).
 * From LK_SUM_KERNEL on, b1 / b2 follow k_lk_ring's two paths: an iteration whose vote passes takes the exact path
 * (the ten b chain totals as integers, combined in float as tail + ((c0 + c2) + (c1 + c3))), any other takes the float
 * chains; after the first rejected iteration of a level-solve the rest of it replays, as in the kernel.  LK_SUM_KERNEL
 * is the kernel's rule and must equal mode 0; LK_SUM_M1..M6 are wrong rules that tests use to show the LK sum-edge
 * fixture notices one. */
enum {
    LK_SUM_CV2 = 0,         /* cv2's order: (q0 + q2) + (q1 + q3) lane reduction                                  */
    LK_SUM_SEQ = 1,         /* lane reduction ((q0 + q1) + q2) + q3                                               */
    LK_SUM_PAIRS = 2,       /* lane reduction (q0 + q1) + (q2 + q3)                                               */
    LK_SUM_SCALAR = 9,      /* no SIMD body: every column in the scalar chain                                     */
    LK_SUM_KERNEL = 10,     /* vote max(P, N) <= 2^24 on all ten chains (sum |product| + |total| <= 2^25)           */
    LK_SUM_M1 = 11,         /* vote max(P, N) <= 2^25 (twice too permissive)                                       */
    LK_SUM_M2 = 12,         /* vote sum |product| <= 2^25, without the sign term                                   */
    LK_SUM_M3 = 13,         /* the vote ignores the two tail chains                                                */
    LK_SUM_M4 = 14,         /* the vote ignores b2's five chains                                                   */
    LK_SUM_M5 = 15,         /* the exact path combines (c0 + c1) + (c2 + c3)                                       */
    LK_SUM_M6 = 16,         /* the replay adds the tail chain column-major                                         */
    /* From LK_SUM_WIN on, b1 / b2 are formed by lk_win_b, k_lk_win's chains (no vote, no exact path).  LK_SUM_WIN is that
     * kernel's rule and must equal mode 0; the others change one piece of it, so that tests can show the LK window-edge
     * fixture notices each change. */
    LK_SUM_WIN = 17,        /* k_lk_win's rule                                                                     */
    LK_SUM_TAILCOL = 18,    /* the b tail chains add column-major                                                  */
    LK_SUM_SIMD4 = 19,      /* a 4-wide SIMD split nsimd = W & ~3 (A and b; a b column without a partner x + 4 < nsimd
                             * is added alone)                                                                      */
    LK_SUM_ADJ = 20,        /* b chain q adds the pair sums of columns (x, x + 1), x = 2q + 8m, not (x, x + 4)       */
    LK_SUM_COMBINE = 21,    /* the chain totals of A and b combine as (c0 + c1) + (c2 + c3)                        */
};
static int g_sum_mode = 0;
void lk_set_sum_mode(int m) { g_sum_mode = m; }

/* The ten b chains of one Newton iteration (b1 chains 0..3, b1 tail, b2 chains 0..3, b2 tail), split as k_lk_ring
 * splits them: a SIMD chain q holds the products of columns x = q (mod 4), x < nsimd, and adds them in pairs (x, x+4)
 * row by row; the tail holds columns nsimd.. row-major. */
typedef struct {
    int64_t sabs[10];       /* sum |product|                                                                      */
    int64_t pos[10];        /* P: sum of the positive products                                                    */
    int64_t neg[10];        /* N: sum of |negative products|                                                      */
    int64_t total[10];      /* P - N                                                                              */
    int64_t maxpre[10];     /* largest |prefix sum| in cv2's chain order                                          */
    int64_t maxadd[10];     /* largest |addend| (a pair sum in the SIMD chains, a product in the tail)            */
    float tail_colmajor[2]; /* the tail chains added column-major in float (LK_SUM_M6)                            */
} lk_chains_t;

static void lk_chain_info(const int *diffs_all, const int16_t *dIbuf, int win, lk_chains_t *c)
{
    const int nsimd = (win / 8) * 8;
    memset(c, 0, sizeof(*c));
    for (int comp = 0; comp < 2; comp++) {
        for (int q = 0; q < 5; q++) {
            const int k = comp * 5 + q;
            long long pre = 0;
            for (int y = 0; y < win; y++) {
                const int *d = diffs_all + y * win;
                const int16_t *g = dIbuf + y * win * 2 + comp;
                if (q < 4) {
                    for (int x0 = q; x0 < nsimd; x0 += 8) {
                        long long v0 = (long long)d[x0] * g[2 * x0], v1 = (long long)d[x0 + 4] * g[2 * (x0 + 4)];
                        long long pair = v0 + v1;
                        c->pos[k] += (v0 > 0 ? v0 : 0) + (v1 > 0 ? v1 : 0);
                        c->neg[k] += (v0 < 0 ? -v0 : 0) + (v1 < 0 ? -v1 : 0);
                        pre += pair;
                        if (llabs(pre) > c->maxpre[k]) c->maxpre[k] = llabs(pre);
                        if (llabs(pair) > c->maxadd[k]) c->maxadd[k] = llabs(pair);
                    }
                } else {
                    for (int x = nsimd; x < win; x++) {
                        long long v = (long long)d[x] * g[2 * x];
                        c->pos[k] += v > 0 ? v : 0;
                        c->neg[k] += v < 0 ? -v : 0;
                        pre += v;
                        if (llabs(pre) > c->maxpre[k]) c->maxpre[k] = llabs(pre);
                        if (llabs(v) > c->maxadd[k]) c->maxadd[k] = llabs(v);
                    }
                }
            }
            c->sabs[k] = c->pos[k] + c->neg[k];
            c->total[k] = pre;
        }
        float t = 0.f;
        for (int x = nsimd; x < win; x++)
            for (int y = 0; y < win; y++)
                t += (float)(diffs_all[y * win + x] * dIbuf[(y * win + x) * 2 + comp]);
        c->tail_colmajor[comp] = t;
    }
}

/* k_lk_ring's vote (mode LK_SUM_KERNEL) or a wrong one (LK_SUM_M1..M4): may this iteration take the exact path?
 * Every prefix of a chain lies in [-N, P], so max(P, N) <= 2^24 makes each one an exact float. */
static int lk_vote(const lk_chains_t *c, int mode)
{
    const long long LIM = 1LL << 24;
    for (int k = 0; k < 10; k++) {
        if (mode == LK_SUM_M3 && (k == 4 || k == 9)) continue;
        if (mode == LK_SUM_M4 && k >= 5) continue;
        const long long P = c->pos[k], N = c->neg[k];
        const int ok = mode == LK_SUM_M1 ? (P <= 2 * LIM && N <= 2 * LIM)
                     : mode == LK_SUM_M2 ? (P + N <= 2 * LIM)
                     : (P <= LIM && N <= LIM);
        if (!ok) return 0;
    }
    return 1;
}

/* the exact path's float combination of one quantity's chain totals t[0..3] and tail t[4] */
static float lk_exact_combine(const int64_t *t, int mode)
{
    const float c0 = (float)t[0], c1 = (float)t[1], c2 = (float)t[2], c3 = (float)t[3];
    const float simd = mode == LK_SUM_M5 ? (c0 + c1) + (c2 + c3) : (c0 + c2) + (c1 + c3);
    return (float)t[4] + simd;
}

/* Optional bookkeeping for kernel design (not part of the checker): how often are all partial sums of the b chains
 * exactly representable?  [0] iterations, [1] sum|addend| <= 2^24 on every chain (the kernel's former test),
 * [2] strip bound: sum over the kernel's strips of max|running strip sum| <= 2^24 and every addend <= 2^24,
 * [3] truth: every chain prefix and every addend <= 2^24 in magnitude,
 * [4] sign split: max(P, N) <= 2^24 on every chain (the vote k_lk_ring runs),
 * [5] iterations the sign split accepts although a prefix or an addend leaves +-2^24 (0 if the vote is sound). */
static long long g_stats[8];
static int g_stats_on = 0;
void lk_stats_enable(int on) { g_stats_on = on; for (int i = 0; i < 8; i++) g_stats[i] = 0; }
void lk_stats_get(long long *out) { for (int i = 0; i < 8; i++) out[i] = g_stats[i]; }

static void lk_chain_stats(const int *diffs_all, const int16_t *dIbuf, int win, const lk_chains_t *ch)
{
    /* diffs_all: win x win residuals; dIbuf: win x win x 2 gradients */
    const long long LIM = 1LL << 24;
    int ok_old = 1, ok_strip = 1, ok_true = 1;
    for (int comp = 0; comp < 2; comp++) {
        /* SIMD chains q = 0..3: per row the pairs (q, q+4) then (q+8, q+12) */
        for (int q = 0; q < 4; q++) {
            long long sabs = 0, pre = 0, maxpre = 0, maxadd = 0;
            for (int y = 0; y < win; y++)
                for (int g = 0; g < 2; g++) {
                    int x0 = q + 8 * g, x1 = x0 + 4;
                    long long v0 = (long long)diffs_all[y * win + x0] * dIbuf[(y * win + x0) * 2 + comp];
                    long long v1 = (long long)diffs_all[y * win + x1] * dIbuf[(y * win + x1) * 2 + comp];
                    long long pair = v0 + v1;
                    sabs += llabs(v0) + llabs(v1);
                    pre += pair;
                    if (llabs(pre) > maxpre) maxpre = llabs(pre);
                    if (llabs(pair) > maxadd) maxadd = llabs(pair);
                }
            if (sabs > LIM) ok_old = 0;
            if (maxpre > LIM || maxadd > LIM) ok_true = 0;
            /* strip bound: strips (col, rows 0..10) and (col, rows 11..20) of the chain's 4 columns */
            long long bound = 0, maxa = 0;
            for (int c = q; c < 16; c += 4)
                for (int half = 0; half < 2; half++) {
                    long long run = 0, mx = 0;
                    for (int y = half ? 11 : 0; y < (half ? win : 11); y++) {
                        long long v = (long long)diffs_all[y * win + c] * dIbuf[(y * win + c) * 2 + comp];
                        run += v;
                        if (llabs(run) > mx) mx = llabs(run);
                        if (llabs(v) > maxa) maxa = llabs(v);
                    }
                    bound += mx;
                }
            if (bound > LIM || 2 * maxa > LIM) ok_strip = 0;
        }
        /* tail chain: columns 16..20 row-major */
        {
            long long sabs = 0, pre = 0, maxpre = 0, maxadd = 0;
            for (int y = 0; y < win; y++)
                for (int x = 16; x < win; x++) {
                    long long v = (long long)diffs_all[y * win + x] * dIbuf[(y * win + x) * 2 + comp];
                    sabs += llabs(v); pre += v;
                    if (llabs(pre) > maxpre) maxpre = llabs(pre);
                    if (llabs(v) > maxadd) maxadd = llabs(v);
                }
            if (sabs > LIM) ok_old = 0;
            if (maxpre > LIM || maxadd > LIM) ok_true = 0;
            static const int seg_r0[6] = {0, 4, 8, 12, 15, 18}, seg_n[6] = {4, 4, 4, 3, 3, 3};
            long long bound = 0;
            for (int x = 16; x < win; x++)
                for (int sg = 0; sg < 6; sg++) {
                    long long run = 0, mx = 0;
                    for (int y = seg_r0[sg]; y < seg_r0[sg] + seg_n[sg]; y++) {
                        run += (long long)diffs_all[y * win + x] * dIbuf[(y * win + x) * 2 + comp];
                        if (llabs(run) > mx) mx = llabs(run);
                    }
                    bound += mx;
                }
            if (bound > LIM || maxadd > LIM) ok_strip = 0;
        }
    }
    const int ok_sign = lk_vote(ch, LK_SUM_KERNEL);
    g_stats[0]++; g_stats[1] += ok_old; g_stats[2] += ok_strip; g_stats[3] += ok_true;
    g_stats[4] += ok_sign; g_stats[5] += ok_sign && !ok_true;
}

/* Optional per-point event log (off by default; tests/test_oracle_lk_edges.py and tests/golden/make_lk_edges.py read it
 * to find and check the inputs that sit on the decision edges of a level-solve).  One record per level-solve set-up
 * (minEig, D, the I window origin) and one per Newton iteration (the step, the half-step sums, the J window origin,
 * ||delta||^2 in double and in float, and per b chain as k_lk_ring splits them: sum |product|, P and N, the signed
 * total, the largest |prefix| and |addend| in cv2's order and the float32 chain as cv2 adds it), plus one for the
 * level-0 final re-check when it clears the status.  The layout is mirrored by oracle/cref.py:LK_EVENT. */
enum {
    LK_EV_ITER = 0,     /* an iteration after which the solve goes on                                   */
    LK_EV_EPS = 1,      /* ended by delta.ddot(delta) <= eps^2                                          */
    LK_EV_HALF = 2,     /* ended by |dx + pdx| < 0.01 && |dy + pdy| < 0.01 (the half-step exit)         */
    LK_EV_CAP = 3,      /* the max_count-th iteration, none of the exits taken                          */
    LK_EV_JOUT = 4,     /* the J window left the image before iteration `iter` (no step computed)       */
    LK_EV_SETUP = 5,    /* level-solve set up: minEig >= threshold and D >= FLT_EPSILON                 */
    LK_EV_REJECT = 6,   /* level-solve rejected: minEig < threshold or D < FLT_EPSILON                  */
    LK_EV_IOUT = 7,     /* the I window is out of the image: the level is skipped                       */
    LK_EV_FINAL = 8,    /* level 0 final re-check: the end position's window is out of the image        */
};
typedef struct {
    int32_t pt, level, iter, kind;
    float min_eig, D, dx, dy, sdx, sdy;     /* sdx = dx + pdx, sdy = dy + pdy (pdx = pdy = 0 at iteration 0) */
    int32_t ipx, ipy, inx, iny;             /* floored window origins: I (level set-up), J (this iteration)  */
    double d2;                              /* (double)dx*dx + (double)dy*dy                                  */
    float d2f;                              /* dx*dx + dy*dy in float                                         */
    int32_t pad_;
    int64_t sabs[10];                       /* b1 chains 0..3, b1 tail, b2 chains 0..3, b2 tail: sum |product| */
    int64_t pos[10], neg[10], total[10];    /* P, N, P - N (lk_chains_t)                                      */
    int64_t maxpre[10], maxadd[10];         /* largest |prefix|, |addend| in cv2's chain order                */
    float fchain[10];                       /* the chain's float32 sum as cv2 forms it                        */
} lk_event_t;
static lk_event_t *g_log = NULL;
static long long g_log_cap = 0, g_log_n = 0;
void lk_log_enable(void *buf, long long cap) { g_log = (lk_event_t *)buf; g_log_cap = buf ? cap : 0; g_log_n = 0; }
long long lk_log_count(void) { return g_log_n; }
int lk_log_record_size(void) { return (int)sizeof(lk_event_t); }

static lk_event_t *lk_log_add(int pt, int level, int iter, int kind)
{
    static lk_event_t sink;
    lk_event_t *e = g_log_n < g_log_cap ? &g_log[g_log_n] : &sink;    /* counted even when full: the caller re-runs */
    g_log_n++;
    memset(e, 0, sizeof(*e));
    e->pt = pt; e->level = level; e->iter = iter; e->kind = kind;
    return e;
}

static inline float reduce4(const float q[4])
{
    switch (g_sum_mode) {
    default:
    case 0: return (q[0] + q[2]) + (q[1] + q[3]);   /* SSE v_reduce_sum: movehl + shuffle */
    case 1: return ((q[0] + q[1]) + q[2]) + q[3];
    case 2: case LK_SUM_COMBINE: return (q[0] + q[1]) + (q[2] + q[3]);
    }
}

/* b1 (comp 0) or b2 (comp 1) as k_lk_win forms them in mode LK_SUM_WIN: SIMD chain q adds, row by row, the float of the
 * integer pair sum of columns (x, x + 4), x = q + 8m < nsimd; the tail adds the products of columns nsimd.. row-major;
 * the total is tail + ((c0 + c2) + (c1 + c3)).  The modes after it change one piece (see LK_SUM_*). */
static float lk_win_b(const int *d, const int16_t *g, int win, int comp, int mode)
{
    const int nsimd = mode == LK_SUM_SIMD4 ? (win & ~3) : (win / 8) * 8;
    float c[4] = {0.f, 0.f, 0.f, 0.f}, t = 0.f;
    for (int y = 0; y < win; y++) {
        const int *dr = d + y * win;
        const int16_t *gr = g + y * win * 2 + comp;
        for (int q = 0; q < 4; q++) {
            if (mode == LK_SUM_ADJ) {
                for (int x = 2 * q; x < nsimd; x += 8)
                    c[q] += (float)(dr[x] * gr[2 * x] + dr[x + 1] * gr[2 * (x + 1)]);
            } else {
                for (int x = q; x < nsimd; x += 8)
                    c[q] += (float)(dr[x] * gr[2 * x] + (x + 4 < nsimd ? dr[x + 4] * gr[2 * (x + 4)] : 0));
            }
        }
        if (mode != LK_SUM_TAILCOL)
            for (int x = nsimd; x < win; x++) t += (float)(dr[x] * gr[2 * x]);
    }
    if (mode == LK_SUM_TAILCOL)
        for (int x = nsimd; x < win; x++)
            for (int y = 0; y < win; y++) t += (float)(d[y * win + x] * g[(y * win + x) * 2 + comp]);
    const float simd = mode == LK_SUM_COMBINE ? (c[0] + c[1]) + (c[2] + c[3]) : (c[0] + c[2]) + (c[1] + c[3]);
    return t + simd;
}

#define W_BITS 14
#define DESCALE(x, n) (((x) + (1 << ((n) - 1))) >> (n))

static inline int cv_floor(float v) { return (int)floorf(v); }
static inline int cv_round(float v) { return (int)lrintf(v); } /* round-half-even */

/*
 * One calcOpticalFlowPyrLK call, flags = 0, err requested.
 * next_pts is output only (no OPTFLOW_USE_INITIAL_FLOW).
 * iters_out (optional): total J-iterations per point, for workload statistics.
 */
void lk_track(const lk_pyr_t *prev, const lk_pyr_t *next,
              const float *prev_pts, float *next_pts, uint8_t *status, float *err,
              int npts, int win, int max_count, double epsilon, double min_eig_thr,
              int *iters_out)
{
    int nlev = prev->nlevels < next->nlevels ? prev->nlevels : next->nlevels;
    int max_level = nlev - 1;
    const float half = (win - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (1 << 20);
    /* calcOpticalFlowPyrLK clamps the criteria (maxCount to [0, 100], epsilon to [0, 10]), and LKTrackerInvoker keeps
     * minEigThreshold as a float: minEig is compared with the float threshold, in float */
    if (max_count < 0) max_count = 0; if (max_count > 100) max_count = 100;
    if (epsilon < 0.) epsilon = 0.; if (epsilon > 10.) epsilon = 10.;
    double eps2 = epsilon * epsilon;
    const float min_eig_f = (float)min_eig_thr;
    int16_t *Ibuf = (int16_t *)malloc(sizeof(int16_t) * win * win * 3);
    int16_t *dIbuf = Ibuf + win * win;
    /* columns handled by the 8-wide SIMD body (LK_SUM_SIMD4: a wrong 4-wide split) */
    const int nsimd = g_sum_mode == LK_SUM_SIMD4 ? (win & ~3) : (win / 8) * 8;

    for (int i = 0; i < npts; i++) { status[i] = 1; if (err) err[i] = 0.f; if (iters_out) iters_out[i] = 0; }

    for (int level = max_level; level >= 0; level--) {
        const lk_level_t *I = &prev->lv[level], *J = &next->lv[level];
        const uint8_t *Ibase = I->img + I->pad * I->istep + I->pad;
        const uint8_t *Jbase = J->img + J->pad * J->istep + J->pad;
        const int16_t *Dbase = I->deriv + I->pad * I->dstep + 2 * I->pad;
        for (int pi = 0; pi < npts; pi++) {
            float px = prev_pts[2 * pi] * (float)(1. / (1 << level));
            float py = prev_pts[2 * pi + 1] * (float)(1. / (1 << level));
            float nx, ny;
            if (level == max_level) { nx = px; ny = py; }
            else { nx = next_pts[2 * pi] * 2.f; ny = next_pts[2 * pi + 1] * 2.f; }
            next_pts[2 * pi] = nx; next_pts[2 * pi + 1] = ny;

            px -= half; py -= half;
            int ipx = cv_floor(px), ipy = cv_floor(py);
            if (ipx < -win || ipx >= I->w || ipy < -win || ipy >= I->h) {
                if (g_log) { lk_event_t *e = lk_log_add(pi, level, -1, LK_EV_IOUT); e->ipx = ipx; e->ipy = ipy; }
                if (level == 0) { status[pi] = 0; if (err) err[pi] = 0.f; }
                continue;
            }
            float a = px - ipx, b = py - ipy;
            int iw00 = cv_round((1.f - a) * (1.f - b) * (1 << W_BITS));
            int iw01 = cv_round(a * (1.f - b) * (1 << W_BITS));
            int iw10 = cv_round((1.f - a) * b * (1 << W_BITS));
            int iw11 = (1 << W_BITS) - iw00 - iw01 - iw10;

            float qA11[4] = {0, 0, 0, 0}, qA12[4] = {0, 0, 0, 0}, qA22[4] = {0, 0, 0, 0};
            float iA11 = 0, iA12 = 0, iA22 = 0;
            for (int y = 0; y < win; y++) {
                const uint8_t *src = Ibase + (y + ipy) * I->istep + ipx;
                const int16_t *dsrc = Dbase + (y + ipy) * I->dstep + 2 * ipx;
                int16_t *Ip = Ibuf + y * win, *dIp = dIbuf + y * win * 2;
                for (int x = 0; x < win; x++, dsrc += 2, dIp += 2) {
                    int ival = DESCALE(src[x] * iw00 + src[x + 1] * iw01 +
                                       src[x + I->istep] * iw10 + src[x + I->istep + 1] * iw11, W_BITS - 5);
                    int ixval = DESCALE(dsrc[0] * iw00 + dsrc[2] * iw01 +
                                        dsrc[I->dstep] * iw10 + dsrc[I->dstep + 2] * iw11, W_BITS);
                    int iyval = DESCALE(dsrc[1] * iw00 + dsrc[3] * iw01 +
                                        dsrc[I->dstep + 1] * iw10 + dsrc[I->dstep + 3] * iw11, W_BITS);
                    Ip[x] = (int16_t)ival; dIp[0] = (int16_t)ixval; dIp[1] = (int16_t)iyval;
                    float fx = (float)ixval, fy = (float)iyval;
                    if (x < nsimd && g_sum_mode != 9) {
                        int l = x & 3;
                        /* v_muladd without FMA: separately rounded mul and add */
                        qA22[l] = fy * fy + qA22[l];
                        qA12[l] = fx * fy + qA12[l];
                        qA11[l] = fx * fx + qA11[l];
                    } else {
                        iA11 += (float)(ixval * ixval);
                        iA12 += (float)(ixval * iyval);
                        iA22 += (float)(iyval * iyval);
                    }
                }
            }
            if (g_sum_mode != 9) {
                iA11 += reduce4(qA11); iA12 += reduce4(qA12); iA22 += reduce4(qA22);
            }
            float A11 = iA11 * FLT_SCALE, A12 = iA12 * FLT_SCALE, A22 = iA22 * FLT_SCALE;
            float D = A11 * A22 - A12 * A12;
            float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (2 * win * win);
            if (g_log) {
                lk_event_t *e = lk_log_add(pi, level, -1, (minEig < min_eig_f || D < FLT_EPSILON) ? LK_EV_REJECT : LK_EV_SETUP);
                e->min_eig = minEig; e->D = D; e->ipx = ipx; e->ipy = ipy;
            }
            if (minEig < min_eig_f || D < FLT_EPSILON) {
                if (level == 0) status[pi] = 0;
                continue;
            }
            D = 1.f / D;

            float npx = nx - half, npy = ny - half;
            float pdx = 0, pdy = 0;
            int replayed = 0;
            for (int j = 0; j < max_count; j++) {
                int inx = cv_floor(npx), iny = cv_floor(npy);
                if (inx < -win || inx >= J->w || iny < -win || iny >= J->h) {
                    if (g_log) {
                        lk_event_t *e = lk_log_add(pi, level, j, LK_EV_JOUT);
                        e->min_eig = minEig; e->ipx = ipx; e->ipy = ipy; e->inx = inx; e->iny = iny;
                    }
                    if (level == 0) status[pi] = 0;
                    break;
                }
                if (iters_out) iters_out[pi]++;
                a = npx - inx; b = npy - iny;
                iw00 = cv_round((1.f - a) * (1.f - b) * (1 << W_BITS));
                iw01 = cv_round(a * (1.f - b) * (1 << W_BITS));
                iw10 = cv_round((1.f - a) * b * (1 << W_BITS));
                iw11 = (1 << W_BITS) - iw00 - iw01 - iw10;
                float qb0[4] = {0, 0, 0, 0}, qb1[4] = {0, 0, 0, 0};
                float ib1 = 0, ib2 = 0;
                int diffs_all[32 * 32];
                for (int y = 0; y < win; y++) {
                    const uint8_t *Jp = Jbase + (y + iny) * J->istep + inx;
                    const int16_t *Ip = Ibuf + y * win, *dIp = dIbuf + y * win * 2;
                    int *diffs = diffs_all + y * win;
                    for (int x = 0; x < win; x++)
                        diffs[x] = DESCALE(Jp[x] * iw00 + Jp[x + 1] * iw01 +
                                           Jp[x + J->istep] * iw10 + Jp[x + J->istep + 1] * iw11, W_BITS - 5) - Ip[x];
                    int x = 0;
                    if (g_sum_mode != 9) {
                        for (; x <= win - 8; x += 8) {
                            /* lanes: qb0 = [bx(0,4) by(0,4) bx(1,5) by(1,5)], qb1 = [bx(2,6) by(2,6) bx(3,7) by(3,7)] */
                            for (int l = 0; l < 4; l++) {
                                int p0 = x + l, p1 = x + l + 4;
                                int sx = dIp[2 * p0] * diffs[p0] + dIp[2 * p1] * diffs[p1];
                                int sy = dIp[2 * p0 + 1] * diffs[p0] + dIp[2 * p1 + 1] * diffs[p1];
                                float *q = (l < 2) ? qb0 : qb1;
                                int li = (l & 1) * 2;
                                q[li] += (float)sx;
                                q[li + 1] += (float)sy;
                            }
                        }
                    }
                    for (; x < win; x++) {
                        ib1 += (float)(diffs[x] * dIp[2 * x]);
                        ib2 += (float)(diffs[x] * dIp[2 * x + 1]);
                    }
                }
                const int kernel_mode = g_sum_mode >= LK_SUM_KERNEL && g_sum_mode <= LK_SUM_M6;
                const int want_chains = g_log || (g_stats_on && win == 21) || kernel_mode;
                lk_chains_t ch;
                if (want_chains) lk_chain_info(diffs_all, dIbuf, win, &ch);
                if (g_stats_on && win == 21) lk_chain_stats(diffs_all, dIbuf, win, &ch);
                /* the float chains as cv2 forms them: SIMD chain q is lane q's bx / by, the tails are ib1 / ib2 so far */
                float fchain[10];
                for (int q = 0; q < 4; q++) {
                    const float *qq = (q < 2) ? qb0 : qb1;
                    fchain[q] = qq[(q & 1) * 2]; fchain[5 + q] = qq[(q & 1) * 2 + 1];
                }
                fchain[4] = ib1; fchain[9] = ib2;
                if (g_sum_mode == LK_SUM_M6) { ib1 = ch.tail_colmajor[0]; ib2 = ch.tail_colmajor[1]; }
                if (g_sum_mode != 9) {
                    /* qf0 = interleave_pairs(qb0+qb1) low half = [s0, s2, 0, 0], qf1 = [s1, s3, 0, 0] */
                    float s[4];
                    for (int l = 0; l < 4; l++) s[l] = qb0[l] + qb1[l];
                    float qf0[4] = {s[0], s[2], 0.f, 0.f}, qf1[4] = {s[1], s[3], 0.f, 0.f};
                    ib1 += reduce4(qf0);
                    ib2 += reduce4(qf1);
                }
                if (g_sum_mode >= LK_SUM_WIN) {
                    ib1 = lk_win_b(diffs_all, dIbuf, win, 0, g_sum_mode);
                    ib2 = lk_win_b(diffs_all, dIbuf, win, 1, g_sum_mode);
                }
                if (kernel_mode) {
                    if (!replayed && lk_vote(&ch, g_sum_mode)) {
                        ib1 = lk_exact_combine(ch.total, g_sum_mode);
                        ib2 = lk_exact_combine(ch.total + 5, g_sum_mode);
                    } else {
                        replayed = 1;       /* k_lk_ring replays the rest of the level-solve without a vote */
                    }
                }
                float b1 = ib1 * FLT_SCALE, b2 = ib2 * FLT_SCALE;
                float dx = (float)((A12 * b2 - A22 * b1) * D);
                float dy = (float)((A12 * b1 - A11 * b2) * D);
                npx += dx; npy += dy;
                next_pts[2 * pi] = npx + half; next_pts[2 * pi + 1] = npy + half;
                lk_event_t *ev = NULL;
                if (g_log) {
                    ev = lk_log_add(pi, level, j, j == max_count - 1 ? LK_EV_CAP : LK_EV_ITER);
                    ev->min_eig = minEig; ev->D = D; ev->dx = dx; ev->dy = dy; ev->sdx = dx + pdx; ev->sdy = dy + pdy;
                    ev->ipx = ipx; ev->ipy = ipy; ev->inx = inx; ev->iny = iny;
                    ev->d2 = (double)dx * dx + (double)dy * dy; ev->d2f = dx * dx + dy * dy;
                    memcpy(ev->sabs, ch.sabs, sizeof ch.sabs);
                    memcpy(ev->pos, ch.pos, sizeof ch.pos);
                    memcpy(ev->neg, ch.neg, sizeof ch.neg);
                    memcpy(ev->total, ch.total, sizeof ch.total);
                    memcpy(ev->maxpre, ch.maxpre, sizeof ch.maxpre);
                    memcpy(ev->maxadd, ch.maxadd, sizeof ch.maxadd);
                    memcpy(ev->fchain, fchain, sizeof fchain);
                }
                if ((double)dx * dx + (double)dy * dy <= eps2) { if (ev) ev->kind = LK_EV_EPS; break; }
                if (j > 0 && fabs(dx + pdx) < 0.01 && fabs(dy + pdy) < 0.01) {
                    if (ev) ev->kind = LK_EV_HALF;
                    next_pts[2 * pi] -= dx * 0.5f;
                    next_pts[2 * pi + 1] -= dy * 0.5f;
                    break;
                }
                pdx = dx; pdy = dy;
            }

            if (status[pi] && err && level == 0) {
                float fx = next_pts[2 * pi] - half, fy = next_pts[2 * pi + 1] - half;
                int inx = cv_floor(fx), iny = cv_floor(fy);
                if (inx < -win || inx >= J->w || iny < -win || iny >= J->h) {
                    if (g_log) { lk_event_t *e = lk_log_add(pi, 0, -1, LK_EV_FINAL); e->inx = inx; e->iny = iny; }
                    status[pi] = 0;
                    continue;
                }
                float aa = fx - inx, bb = fy - iny;
                iw00 = cv_round((1.f - aa) * (1.f - bb) * (1 << W_BITS));
                iw01 = cv_round(aa * (1.f - bb) * (1 << W_BITS));
                iw10 = cv_round((1.f - aa) * bb * (1 << W_BITS));
                iw11 = (1 << W_BITS) - iw00 - iw01 - iw10;
                float errval = 0.f;
                for (int y = 0; y < win; y++) {
                    const uint8_t *Jp = Jbase + (y + iny) * J->istep + inx;
                    const int16_t *Ip = Ibuf + y * win;
                    for (int x = 0; x < win; x++) {
                        int diff = DESCALE(Jp[x] * iw00 + Jp[x + 1] * iw01 +
                                           Jp[x + J->istep] * iw10 + Jp[x + J->istep + 1] * iw11, W_BITS - 5) - Ip[x];
                        errval += fabsf((float)diff);
                    }
                }
                err[pi] = errval * 1.f / (32 * win * win);
            }
        }
    }
    free(Ibuf);
}
