// rectify.cu -- rectification of raw stereo frames (include/vo_b200.h, "rectification"): ORB-SLAM2's stereo driver runs
// cv::initUndistortRectifyMap(K, D, R, P, size, CV_32F) once per camera and cv::remap(INTER_LINEAR) on every image.
//
//   * vo_rectify_maps restates initUndistortRectifyMap(CV_32FC1) in double, in the operation order of the build cv2
//     runs on x86-64 CPUs with AVX2 (its dispatched path): iR = inv(P * R) by the cofactor formula cv::invert(DECOMP_LU)
//     uses for 3 x 3 matrices; per row _x, _y, _w from the row index, advanced by 8 * iR's first column per step of 8
//     pixels (pixel l of a step at _x + ir[0] * l), the 8-coefficient rational model with fused multiply-adds where that
//     build has them, and the row's last w % 8 pixels by cv2's scalar loop (a running sum per pixel).  The maps come out
//     as cv2's float bits.
//   * the float maps go to the device once, in the fixed-point form cv::remap makes of them (rint(map * 32), integer part
//     saturated to int16, 5-bit fractions; remap_math.cuh), so the ingest kernel does integer arithmetic only.
#include "ctx.h"
#include <math.h>
#include <string.h>
#include <vector>

namespace {

// the refusals of vo_rectify_maps for one camera: nullptr when it is accepted, else why not
const char* rect_invalid(const vo_rectify_cam* c)
{
    if (c->n_d != 4 && c->n_d != 5 && c->n_d != 8) return "n_d must be 4, 5 or 8";
    for (int i = 0; i < 9; i++)
        if (!isfinite(c->K[i]) || !isfinite(c->R[i]) || !isfinite(c->P[i])) return "a non-finite entry in K, R or P";
    for (int i = 0; i < c->n_d; i++)
        if (!isfinite(c->D[i])) return "a non-finite distortion coefficient";
    return nullptr;
}

// inv(P * R) as cv::invert(DECOMP_LU) computes a 3 x 3 inverse; false when the determinant is 0
bool rect_inverse(const vo_rectify_cam* c, double ir[9])
{
    double m[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
            m[3 * i + j] = c->P[3 * i] * c->R[j] + c->P[3 * i + 1] * c->R[3 + j] + c->P[3 * i + 2] * c->R[6 + j];
#define M(i, j) m[3 * (i) + (j)]
    double d = M(0, 0) * (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) - M(0, 1) * (M(1, 0) * M(2, 2) - M(1, 2) * M(2, 0)) +
               M(0, 2) * (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0));
    if (d == 0.0) return false;
    d = 1. / d;
    ir[0] = (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) * d;
    ir[1] = (M(0, 2) * M(2, 1) - M(0, 1) * M(2, 2)) * d;
    ir[2] = (M(0, 1) * M(1, 2) - M(0, 2) * M(1, 1)) * d;
    ir[3] = (M(1, 2) * M(2, 0) - M(1, 0) * M(2, 2)) * d;
    ir[4] = (M(0, 0) * M(2, 2) - M(0, 2) * M(2, 0)) * d;
    ir[5] = (M(0, 2) * M(1, 0) - M(0, 0) * M(1, 2)) * d;
    ir[6] = (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0)) * d;
    ir[7] = (M(0, 1) * M(2, 0) - M(0, 0) * M(2, 1)) * d;
    ir[8] = (M(0, 0) * M(1, 1) - M(0, 1) * M(1, 0)) * d;
#undef M
    return true;
}

// cvRound(v * 32) of a float map value: round half to even; outside the int32 range (or NaN) INT_MIN, as x86's
// cvtss2si returns it
inline int round_fix(float v)
{
    const float s = v * 32.f;
    if (!(fabsf(s) < 2147483648.f)) return INT32_MIN;
    return (int)lrintf(s);
}
inline int16_t sat16(int v) { return (int16_t)(v < -32768 ? -32768 : v > 32767 ? 32767 : v); }

// float maps -> the fixed-point entries cv::remap computes from them
void rect_fixed(const float* mx, const float* my, size_t n, vorect::MapEntry* xy, uint16_t* a)
{
    for (size_t i = 0; i < n; i++) {
        const int X = round_fix(mx[i]), Y = round_fix(my[i]);
        xy[i].x = sat16(X >> 5);
        xy[i].y = sat16(Y >> 5);
        a[i] = (uint16_t)((Y & 31) * 32 + (X & 31));
    }
}

// bytes of one camera's fixed maps at n pixels: the MapEntry plane, then the fractions (each 256-byte aligned)
inline size_t rect_xy_bytes(size_t n) { return (n * sizeof(vorect::MapEntry) + 255) & ~(size_t)255; }
inline size_t rect_a_bytes(size_t n) { return (n * sizeof(uint16_t) + 255) & ~(size_t)255; }

}  // namespace

// one step of cv2's vectorised loop (its AVX2 build: v_muladd is a fused multiply-add) for the pixel at x / y / w
// before the division by w: returns u, v in double
static inline void rect_simd_px(double x, double y, double ww, const double* d, double fx, double fy, double u0, double v0,
                                double* u, double* v)
{
    const double k1 = d[0], k2 = d[1], p1 = d[2], p2 = d[3], k3 = d[4], k4 = d[5], k5 = d[6], k6 = d[7];
    const double m2 = 1.0 / ww;
    x = x * m2; y = y * m2;
    double xd = x * x, yd = y * y;
    const double r2 = xd + yd;
    double m0 = fma(fma(fma(k3, r2, k2), r2, k1), r2, 1.0);
    m0 = m0 / fma(fma(fma(k6, r2, k5), r2, k4), r2, 1.0);
    xd = fma(2.0, xd, r2);
    yd = fma(2.0, yd, r2);
    const double mm = (x * y) * 2.0;
    x = x * m0; y = y * m0;
    xd = fma(xd, p2, x);
    yd = fma(yd, p1, y);
    xd = fma(p1, mm, xd);
    yd = fma(p2, mm, yd);
    // the thin-prism terms (s1..s4 = 0) and the tilt projection (the identity), as the loop applies them
    const double r4 = r2 * r2;
    xd = fma(0.0, r2, fma(0.0, r4, xd));
    yd = fma(0.0, r2, fma(0.0, r4, yd));
    const double X = fma(1.0, xd, fma(0.0, yd, 0.0)), Y = fma(0.0, xd, fma(1.0, yd, 0.0));
    double Z = fma(0.0, xd, fma(0.0, yd, 1.0));
    Z = Z == 0.0 ? 1.0 : 1.0 / Z;
    *u = fma(fx * Z, X, u0);
    *v = fma(fy * Z, Y, v0);
}

extern "C" int vo_rectify_maps(const vo_rectify_cam* c, int w, int h, float* map_x, float* map_y)
{
    if (!c || !map_x || !map_y || w <= 0 || h <= 0 || rect_invalid(c)) return VO_E_INVALID;
    double ir[9];
    if (!rect_inverse(c, ir)) return VO_E_INVALID;
    const double u0 = c->K[2], v0 = c->K[5], fx = c->K[0], fy = c->K[4];
    double d[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < c->n_d; i++) d[i] = c->D[i];
    const double k1 = d[0], k2 = d[1], p1 = d[2], p2 = d[3], k3 = d[4], k4 = d[5], k5 = d[6], k6 = d[7];
    // the vectorised loop's lane offsets: pixel j0 + l of a step reads _x + ir[0] * l (l < 8)
    constexpr int STEP = 8;
    double sx[STEP], sy[STEP], sw[STEP];
    for (int l = 0; l < STEP; l++) { sx[l] = ir[0] * l; sy[l] = ir[3] * l; sw[l] = ir[6] * l; }
    for (int i = 0; i < h; i++) {
        float* mx = map_x + (size_t)i * w;
        float* my = map_y + (size_t)i * w;
        // (the build contracts these, and the scalar loop's expressions below, into fused multiply-adds)
        double _x = fma((double)i, ir[1], ir[2]), _y = fma((double)i, ir[4], ir[5]), _w = fma((double)i, ir[7], ir[8]);
        int j = 0;
        for (; j <= w - STEP; j += STEP, _x += STEP * ir[0], _y += STEP * ir[3], _w += STEP * ir[6])
            for (int l = 0; l < STEP; l++) {
                double u, v;
                rect_simd_px(_x + sx[l], _y + sy[l], _w + sw[l], d, fx, fy, u0, v0, &u, &v);
                mx[j + l] = (float)u;
                my[j + l] = (float)v;
            }
        for (; j < w; j++, _x += ir[0], _y += ir[3], _w += ir[6]) {
            const double ww = 1. / _w, x = _x * ww, y = _y * ww;
            const double x2 = x * x, y2 = y * y;
            const double r2 = x2 + y2, _2xy = 2 * x * y;
            const double kr = fma(fma(fma(k3, r2, k2), r2, k1), r2, 1) / fma(fma(fma(k6, r2, k5), r2, k4), r2, 1);
            const double xd = fma(0. * r2, r2, fma(0., r2, fma(p2, fma(2, x2, r2), fma(p1, _2xy, x * kr))));
            const double yd = fma(0. * r2, r2, fma(0., r2, fma(p2, _2xy, fma(p1, fma(2, y2, r2), y * kr))));
            mx[j] = (float)fma(fx * 1., xd, u0);
            my[j] = (float)fma(fy * 1., yd, v0);
        }
    }
    return VO_OK;
}

int vo_rect_check(vo_ctx* ctx, const char* who, const char* name, const vo_rectify_cam* c)
{
    const char* why = rect_invalid(c);
    double ir[9];
    if (!why && !rect_inverse(c, ir)) why = "P * R is singular";
    if (why) { vo_set_error(ctx, "%s: %s camera: %s", who, name, why); return VO_E_INVALID; }
    return VO_OK;
}

RectMap vo_rect_map(const vo_ctx* ctx, int q, int k, int w, int h)
{
    const size_t n = (size_t)w * h;
    const uint8_t* b = (const uint8_t*)ctx->d_rect[q];
    return RectMap{(const vorect::MapEntry*)(b + k * rect_xy_bytes(n)),
                   (const uint16_t*)(b + 2 * rect_xy_bytes(n) + k * rect_a_bytes(n))};
}

int vo_rect_upload(vo_ctx* ctx, int q, const vo_rectify& r, int w, int h, cudaStream_t st, bool grow_ok)
{
    const size_t n = (size_t)w * h, bytes = 2 * (rect_xy_bytes(n) + rect_a_bytes(n));
    std::vector<float> mx(n), my(n);
    std::vector<uint8_t> host(bytes);
    const vo_rectify_cam* cams[2] = {&r.left, &r.right};
    for (int k = 0; k < 2; k++) {
        if (vo_rectify_maps(cams[k], w, h, mx.data(), my.data())) {     // checked when the setting was made
            vo_set_error(ctx, "rectification maps of sequence %d refused", q);
            return VO_E_INVALID;
        }
        rect_fixed(mx.data(), my.data(), n, (vorect::MapEntry*)(host.data() + k * rect_xy_bytes(n)),
                   (uint16_t*)(host.data() + 2 * rect_xy_bytes(n) + k * rect_a_bytes(n)));
    }
    if (ctx->rect_bytes[q] < bytes) {
        if (ctx->d_rect[q]) {
            if (grow_ok) cudaFree(ctx->d_rect[q]);
            else ctx->rect_dead.push_back(ctx->d_rect[q]);
        }
        ctx->d_rect[q] = nullptr; ctx->rect_bytes[q] = 0;
        VO_CUDA_CHECK(cudaMalloc(&ctx->d_rect[q], bytes));
        ctx->rect_bytes[q] = bytes;
    }
    // a pageable copy: the call returns once the bytes are staged, so `host` may go
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_rect[q], host.data(), bytes, cudaMemcpyHostToDevice, st));
    return VO_OK;
}

extern "C" int vo_remap(vo_ctx* ctx, const uint8_t* src, size_t pitch, int w, int h, const float* map_x, const float* map_y,
                        uint8_t* dst, size_t dst_pitch)
{
    if (!ctx) return VO_E_INVALID;
    if (!src || !map_x || !map_y || !dst || w <= 0 || h <= 0 || pitch < (size_t)w || dst_pitch < (size_t)w) {
        vo_set_error(ctx, "vo_remap: bad argument");
        return VO_E_INVALID;
    }
    { int rcc = vo_claim_buffers(ctx, "vo_remap"); if (rcc) return rcc; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    // scratch (the BGR staging area): source | map entries | fractions | output | descriptor | map table
    const size_t n = (size_t)w * h, up = 256;
    const size_t o_xy = (n + up - 1) / up * up, o_a = o_xy + rect_xy_bytes(n), o_out = o_a + rect_a_bytes(n);
    const size_t o_tab = (o_out + n + up - 1) / up * up, o_map = o_tab + up, bytes = o_map + up;
    int rc = vo_ensure_bgr(ctx, bytes);
    if (rc) return rc;
    uint8_t* b = ctx->d_bgr;
    std::vector<uint8_t> fixed(rect_xy_bytes(n) + rect_a_bytes(n));
    rect_fixed(map_x, map_y, n, (vorect::MapEntry*)fixed.data(), (uint16_t*)(fixed.data() + rect_xy_bytes(n)));
    vo_dimage im{};
    im.data = b; im.row_pitch = (size_t)w; im.pixel_stride = 1; im.channel_stride = 1; im.format = VO_FMT_GRAY;
    const RectMap m{(const vorect::MapEntry*)(b + o_xy), (const uint16_t*)(b + o_a)};
    VO_CUDA_CHECK(cudaMemcpy2DAsync(b, w, src, pitch, w, h, cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(b + o_xy, fixed.data(), fixed.size(), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(b + o_tab, &im, sizeof(im), cudaMemcpyHostToDevice, ctx->stream));
    VO_CUDA_CHECK(cudaMemcpyAsync(b + o_map, &m, sizeof(m), cudaMemcpyHostToDevice, ctx->stream));
    ctx->launches += vo_launch_bgr_to_gray((const vo_dimage*)(b + o_tab), vo_dimage{}, 0, b + o_out, 0, w, h, 1, ctx->stream,
                                           nullptr, (const RectMap*)(b + o_map));
    VO_CUDA_CHECK(cudaGetLastError());
    VO_CUDA_CHECK(cudaMemcpy2DAsync(dst, dst_pitch, b + o_out, w, w, h, cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}

// ---- the sequence modes' settings (host state; the begin and start calls read them, seq_api.cu) --------------------
extern "C" int vo_seq_rectify(vo_ctx* ctx, const vo_rectify* r)
{
    if (!ctx) return VO_E_INVALID;
    int rc;
    if (r && ((rc = vo_rect_check(ctx, "vo_seq_rectify", "left", &r->left)) ||
              (rc = vo_rect_check(ctx, "vo_seq_rectify", "right", &r->right))))
        return rc;
    ctx->rect_single_on = r != nullptr;
    if (r) ctx->rect_single = *r;
    return VO_OK;
}

extern "C" int vo_mseq_rectify(vo_ctx* ctx, int first_slot, int n, const vo_rectify* r)
{
    if (!ctx) return VO_E_INVALID;
    if (first_slot < 0 || n <= 0 || first_slot > VO_MSEQ_MAX - n) {
        vo_set_error(ctx, "vo_mseq_rectify: slots [%d, %d) outside [0, %d)", first_slot, first_slot + n, VO_MSEQ_MAX);
        return VO_E_INVALID;
    }
    for (int i = 0; r && i < n; i++) {
        if (r[i].left.n_d == 0) continue;
        char who[48];
        snprintf(who, sizeof(who), "vo_mseq_rectify: slot %d", first_slot + i);
        int rc;
        if ((rc = vo_rect_check(ctx, who, "left", &r[i].left)) || (rc = vo_rect_check(ctx, who, "right", &r[i].right))) return rc;
    }
    for (int i = 0; i < n; i++) {
        const bool on = r && r[i].left.n_d != 0;
        ctx->slot_rect_on[first_slot + i] = on;
        if (on) ctx->slot_rect[first_slot + i] = r[i];
    }
    return VO_OK;
}
