// remap_math.cuh -- the per-pixel arithmetic of cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) on 8-bit images, shared by
// the ingest kernel (ingest.cu) and its host check (host_check.cpp).
//
// A map entry is the fixed-point form cv::remap makes of float maps (cv::convertMaps(CV_16SC2)): the integer part
// (sx, sy) of rint(map * 32), saturated to int16, and a = (fy << 5) | fx, its two 5-bit fractions.  The four taps
// (sx, sy), (sx + 1, sy), (sx, sy + 1), (sx + 1, sy + 1) are blended with cv2's 15-bit weights
// ((32 - fx) (32 - fy), fx (32 - fy), (32 - fx) fy, fx fy) * 32, which sum to 2^15, and rounded: (sum + 2^14) >> 15.
// A tap outside the image reads 0.  (cv2's table stores 32767 for the weight 32768 of an integer position; for 8-bit
// taps (p * 32767 + 2^14) >> 15 == p, so the two give the same bytes.)
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define VO_HD __host__ __device__ __forceinline__
#else
#define VO_HD inline
#endif

namespace vorect {

struct MapEntry { int16_t x, y; };          // integer part of the source position (cv::convertMaps' CV_16SC2 plane)

// blend of four gray taps at fractions a = (fy << 5) | fx
VO_HD uint8_t blend(int p00, int p01, int p10, int p11, int a)
{
    const int fx = a & 31, fy = a >> 5;
    const int s = (p00 * ((32 - fx) * (32 - fy)) + p01 * (fx * (32 - fy)) + p10 * ((32 - fx) * fy) + p11 * (fx * fy)) * 32;
    return (uint8_t)((s + (1 << 14)) >> 15);
}

// one output pixel from a w x h source: tap(x, y) returns the gray value of an in-image position
template <typename Tap>
VO_HD uint8_t remap_pixel(MapEntry m, int a, int w, int h, const Tap& tap)
{
    const int x0 = m.x, y0 = m.y, x1 = x0 + 1, y1 = y0 + 1;
    const bool cx0 = x0 >= 0 && x0 < w, cx1 = x1 >= 0 && x1 < w, cy0 = y0 >= 0 && y0 < h, cy1 = y1 >= 0 && y1 < h;
    const int p00 = cx0 && cy0 ? tap(x0, y0) : 0, p01 = cx1 && cy0 ? tap(x1, y0) : 0;
    const int p10 = cx0 && cy1 ? tap(x0, y1) : 0, p11 = cx1 && cy1 ? tap(x1, y1) : 0;
    return blend(p00, p01, p10, p11, a);
}

// cv::cvtColor(BGR2GRAY)'s fixed point
VO_HD int gray_of(int b, int g, int r) { return (b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15; }

}  // namespace vorect
