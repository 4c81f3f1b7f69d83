/*
 * oracle/fast_ref.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * Plain-C CPU restatement of cv::FAST(image, keypoints, threshold, nonmaxSuppression)
 * (FastFeatureDetector::TYPE_9_16); the reference's featureDetectionFast() calls it with
 * threshold 20 and non-max suppression (reference src/feature.cpp:39-47).  The arithmetic
 * lives in OpenCV (un-vendored; pinned to 4.13.0 as installed: modules/features2d/src/fast.cpp,
 * fast_score.cpp); the published algorithm is restated here and pinned against cv2 by
 * tests/test_oracle_fast.py (coordinates, raster order and response all identical, at
 * thresholds 0..255 with and without non-max suppression).
 *
 * A pixel p (3-pixel border excluded) is a corner iff >= 9 contiguous pixels of the
 * 16-pixel Bresenham ring are all > p+t or all < p-t.  Its score is the largest t'
 * for which it is still a corner (cornerScore<16>); with non-max suppression a corner
 * is kept iff its score is strictly greater than the scores of its 8 neighbours
 * (non-corners score 0) and its response is the score; without it every corner is
 * kept with response 0.  Output is in raster order.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static const int RING_DX[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
static const int RING_DY[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* largest threshold at which the pixel is still a FAST-9 corner (>= `threshold` if it is one
 * at `threshold`); mirrors cornerScore<16>: result = max(threshold, best arc value) - 1.      */
static int corner_score(const uint8_t *p, int step, int threshold)
{
    int d[25];
    int v = p[0];
    for (int k = 0; k < 25; k++)
        d[k] = v - p[RING_DY[k & 15] * step + RING_DX[k & 15]];
    int a0 = threshold;
    for (int k = 0; k < 16; k += 2) {
        int a = imin(d[k + 1], d[k + 2]);
        a = imin(a, d[k + 3]);
        if (a <= a0) continue;
        a = imin(a, d[k + 4]); a = imin(a, d[k + 5]); a = imin(a, d[k + 6]);
        a = imin(a, d[k + 7]); a = imin(a, d[k + 8]);
        a0 = imax(a0, imin(a, d[k]));
        a0 = imax(a0, imin(a, d[k + 9]));
    }
    int b0 = -a0;
    for (int k = 0; k < 16; k += 2) {
        int b = imax(d[k + 1], d[k + 2]);
        b = imax(b, d[k + 3]); b = imax(b, d[k + 4]); b = imax(b, d[k + 5]);
        if (b >= b0) continue;
        b = imax(b, d[k + 6]); b = imax(b, d[k + 7]); b = imax(b, d[k + 8]);
        b0 = imin(b0, imax(b, d[k]));
        b0 = imin(b0, imax(b, d[k + 9]));
    }
    return -b0 - 1;
}

static int is_corner(const uint8_t *p, int step, int t)
{
    int v = p[0];
    int hi = 0, lo = 0; /* bit k set: ring[k] > v+t / ring[k] < v-t */
    for (int k = 0; k < 16; k++) {
        int r = p[RING_DY[k] * step + RING_DX[k]];
        if (r > v + t) hi |= 1 << k;
        if (r < v - t) lo |= 1 << k;
    }
    for (int pass = 0; pass < 2; pass++) {
        unsigned m = pass ? lo : hi;
        m |= m << 16;
        int run = 0;
        for (int k = 0; k < 32; k++) {
            if (m & (1u << k)) { if (++run >= 9) return 1; }
            else run = 0;
        }
    }
    return 0;
}

/* corner map: 1 for corners; score map: cornerScore for corners, 0 for non-corners.  A corner
 * scores at least the threshold, so at threshold 0 a corner can score 0: whether a pixel is a
 * corner is read from the corner map, never from the score.                                    */
void fast_score_map(const uint8_t *img, int w, int h, int step, int threshold,
                    uint8_t *score /* w*h */, uint8_t *corner /* w*h */)
{
    memset(score, 0, (size_t)w * h);
    memset(corner, 0, (size_t)w * h);
    for (int y = 3; y < h - 3; y++)
        for (int x = 3; x < w - 3; x++) {
            const uint8_t *p = img + y * step + x;
            if (is_corner(p, step, threshold)) {
                corner[y * w + x] = 1;
                score[y * w + x] = (uint8_t)corner_score(p, step, threshold);
            }
        }
}

/* returns number of keypoints; xy (2 floats each) and response are optional outputs.  Without
 * non-max suppression cv::FAST computes no score: every key point then has response 0.          */
int fast_detect(const uint8_t *img, int w, int h, int step, int threshold, int nms,
                float *xy, float *response, int cap)
{
    uint8_t *score = (uint8_t *)malloc((size_t)w * h);
    uint8_t *corner = (uint8_t *)malloc((size_t)w * h);
    fast_score_map(img, w, h, step, threshold, score, corner);
    int n = 0;
    for (int y = 3; y < h - 3; y++)
        for (int x = 3; x < w - 3; x++) {
            if (!corner[y * w + x]) continue;
            int s = score[y * w + x];
            if (nms) {
                /* a score-0 corner (threshold 0) is never strictly greater than all 8 neighbours */
                const uint8_t *q = score + y * w + x;
                if (!(s > q[-1] && s > q[1] && s > q[-w - 1] && s > q[-w] && s > q[-w + 1] &&
                      s > q[w - 1] && s > q[w] && s > q[w + 1]))
                    continue;
            } else {
                s = 0;
            }
            if (n < cap) {
                if (xy) { xy[2 * n] = (float)x; xy[2 * n + 1] = (float)y; }
                if (response) response[n] = (float)s;
            }
            n++;
        }
    free(score);
    free(corner);
    return n;
}
