// pose_math.cuh -- the main loop's pose bookkeeping (src/main.cpp:196-208, src/utils.cpp:57-131) as code that runs on the
// host (pose.cu: vo_pose_integrate, vo_pose_step) and on the device (k_seq_collect: frame_pose of runs begun with
// VO_MSEQ_DEVICE_RESULTS).  Double precision, IEEE operations only (the library builds with -fmad=false, the host code has
// no contraction), so both give the same bits.  The one call that differs is atan2 in the Euler gate: see
// vo_pose_gate_dev.
#pragma once
#include <math.h>

// inverse of T = [R|t; 0 0 0 1] by Gauss-Jordan with partial pivoting (what cv::Mat::inv() defaults to)
__host__ __device__ inline bool vo_invert_rigid4(const double R[9], const double t[3], double inv[16])
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
            if (fabs(a[r][col]) > fabs(a[piv][col])) piv = r;
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

// integrateOdometryStereo: frame_pose *= inv iff 0.05 < |t| < 10.  1 advanced, 0 skipped.
__host__ __device__ inline int vo_integrate_rigid(double frame_pose[16], const double t[3], const double inv[16])
{
    const double scale = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    if (!(scale > 0.05 && scale < 10)) return 0;
    double out[16];
    for (int r = 0; r < 4; r++)
        for (int c = 0; c < 4; c++) {
            double s = 0;
            for (int k = 0; k < 4; k++) s += frame_pose[4 * r + k] * inv[4 * k + c];
            out[4 * r + c] = s;
        }
    for (int i = 0; i < 16; i++) frame_pose[i] = out[i];
    return 1;
}

#ifdef __CUDACC__
// |(float)atan2(y, x)| < 0.1, decided as the host decides it with glibc's atan2 (correctly rounded to double).
// The float of a double a passes iff it is at most 0.099999994f, i.e. iff a <= m = the midpoint of 0.099999994f and 0.1f
// (a tie rounds to the even 0.099999994f).  The double of the exact angle t is at most m iff t <= m + ulp(m) / 2
// (ulp(m) = 2^-56; again a tie rounds to m, whose last bit is even).  The device's atan2 is within 2 ulp of t, so where
// it lies more than 16 ulp from m it decides the same side; in the band between, the angle is compared exactly:
// for x > 0, |t| <= M = m + 2^-57 iff |y| <= x tan(M), with tan(M) as the double-double TH + TL (80 digits, rounded),
// x * TH split exactly with fma, and every other term far below the gap (|y| - x TH is exact by Sterbenz's lemma).
// x <= 0 puts |t| at pi/2 or more, far outside the band; a NaN fails both ways, as on the host.
__device__ inline bool vo_gate_angle_dev(double y, double x)
{
    const double m = 0x1.9999990000000p-4, g = 16 * 0x1p-56;
    const double a = fabs(atan2(y, x));
    if (a <= m - g) return true;
    if (a >= m + g) return false;
    if (!(x > 0)) return false;
    const double TH = 0x1.9af886d90b443p-4, TL = 0x1.4f7ec84a2424fp-58;
    const double ay = fabs(y);
    const double ph = x * TH, pl = __fma_rn(x, TH, -ph);         // x * TH = ph + pl exactly
    const double d = ((ay - ph) - pl) - x * TL;                   // sign of |y| - x tan(M)
    return d <= 0;
}

// vo_pose_step on the device: rotationMatrixToEulerAngles (sy kept in a float, as the reference does), the 0.1 rad gate
// on all three angles, integrateOdometryStereo.  Returns what vo_pose_step returns.
__device__ inline int vo_pose_step_dev(double frame_pose[16], const double R[9], const double t[3])
{
    const float sy = (float)sqrt(R[0] * R[0] + R[3] * R[3]);
    bool ok;
    if (!(sy < 1e-6)) ok = vo_gate_angle_dev(R[7], R[8]) && vo_gate_angle_dev(-R[6], (double)sy) && vo_gate_angle_dev(R[3], R[0]);
    else ok = vo_gate_angle_dev(-R[5], R[4]) && vo_gate_angle_dev(-R[6], (double)sy);      // e[2] = 0
    if (!ok) return 0;
    double inv[16];
    if (!vo_invert_rigid4(R, t, inv)) return -1;                  // VO_E_INVALID, as vo_pose_integrate
    return vo_integrate_rigid(frame_pose, t, inv);
}
#endif
