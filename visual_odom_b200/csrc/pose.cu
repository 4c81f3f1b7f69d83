// pose.cu -- host-side pose bookkeeping of the reference's main loop (SURVEY.md 8f row N2): the Euler-angle gate
// (src/main.cpp:196-203, src/utils.cpp:93-131) and integrateOdometryStereo (src/utils.cpp:57-91).  O(1) per frame,
// double precision, no device work: these are the C-ABI forms the facade's utils.h functions and the streaming
// sequence mode call.
#include "ctx.h"
#include <cmath>
#include <cstring>

extern "C" int vo_pose_is_rotation(const double R[9])
{
    double e = 0;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += R[3 * k + i] * R[3 * k + j];
            const double d = (i == j ? 1.0 : 0.0) - s;
            e += d * d;
        }
    return std::sqrt(e) < 1e-6 ? 1 : 0;
}

extern "C" void vo_pose_euler(const double R[9], float e[3])
{
    // the reference keeps sy in a float and returns a Vec3f
    const float sy = (float)std::sqrt(R[0] * R[0] + R[3] * R[3]);
    if (!(sy < 1e-6)) {
        e[0] = (float)std::atan2(R[7], R[8]);
        e[1] = (float)std::atan2(-R[6], (double)sy);
        e[2] = (float)std::atan2(R[3], R[0]);
    } else {
        e[0] = (float)std::atan2(-R[5], R[4]);
        e[1] = (float)std::atan2(-R[6], (double)sy);
        e[2] = 0.f;
    }
}

// inverse of T = [R|t; 0 0 0 1] by Gauss-Jordan with partial pivoting (what cv::Mat::inv() defaults to)
static bool invert_rigid4(const double R[9], const double t[3], double inv[16])
{
    double a[4][8];
    for (int r = 0; r < 4; r++)
        for (int c = 0; c < 8; c++) a[r][c] = (c >= 4 && c - 4 == r) ? 1.0 : 0.0;
    for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) a[r][c] = R[3 * r + c];
        a[r][3] = t[r];
    }
    a[3][3] = 1.0;
    for (int col = 0; col < 4; col++) {
        int piv = col;
        for (int r = col + 1; r < 4; r++)
            if (std::fabs(a[r][col]) > std::fabs(a[piv][col])) piv = r;
        if (a[piv][col] == 0.0) return false;
        if (piv != col)
            for (int c = 0; c < 8; c++) { const double x = a[piv][c]; a[piv][c] = a[col][c]; a[col][c] = x; }
        const double d = a[col][col];
        for (int c = 0; c < 8; c++) a[col][c] /= d;
        for (int r = 0; r < 4; r++) {
            if (r == col) continue;
            const double f = a[r][col];
            if (f != 0.0)
                for (int c = 0; c < 8; c++) a[r][c] -= f * a[col][c];
        }
    }
    for (int r = 0; r < 4; r++)
        for (int c = 0; c < 4; c++) inv[4 * r + c] = a[r][4 + c];
    return true;
}

extern "C" int vo_pose_integrate(double frame_pose[16], const double R[9], const double t[3], double rigid_inv[16])
{
    double inv[16];
    if (!invert_rigid4(R, t, inv)) return VO_E_INVALID;
    if (rigid_inv) memcpy(rigid_inv, inv, sizeof(inv));
    const double scale = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    if (!(scale > 0.05 && scale < 10)) return 0;
    double out[16];
    for (int r = 0; r < 4; r++)
        for (int c = 0; c < 4; c++) {
            double s = 0;
            for (int k = 0; k < 4; k++) s += frame_pose[4 * r + k] * inv[4 * k + c];
            out[4 * r + c] = s;
        }
    memcpy(frame_pose, out, sizeof(out));
    return 1;
}

extern "C" int vo_pose_step(double frame_pose[16], const double R[9], const double t[3])
{
    float e[3];
    vo_pose_euler(R, e);
    if (!(std::fabs(e[1]) < 0.1 && std::fabs(e[0]) < 0.1 && std::fabs(e[2]) < 0.1)) return 0;   // main.cpp:199
    return vo_pose_integrate(frame_pose, R, t, nullptr);
}

extern "C" int vo_seq_pose(vo_ctx* ctx, double frame_pose[16])
{
    if (!ctx || !ctx->seq_active || !frame_pose) return VO_E_INVALID;
    if (ctx->seq_multi) { vo_set_error(ctx, "vo_seq_pose: the sequences were begun with vo_mseq_begin; use vo_mseq_pose"); return VO_E_INVALID; }
    memcpy(frame_pose, ctx->seq_pose.data(), 16 * sizeof(double));
    return VO_OK;
}
