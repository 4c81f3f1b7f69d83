// pose.cu -- host-side pose bookkeeping of the reference's main loop (SURVEY.md 8f row N2): the Euler-angle gate
// (src/main.cpp:196-203, src/utils.cpp:93-131) and integrateOdometryStereo (src/utils.cpp:57-91).  O(1) per frame,
// double precision, on the host: these are the C-ABI forms the facade's utils.h functions and the streaming sequence
// mode call.  vo_pose_step_device runs the device form (pose_math.cuh, which k_seq_collect integrates frame_pose with)
// on host arrays, for parity tests.
#include "ctx.h"
#include "pose_math.cuh"
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

extern "C" int vo_pose_integrate(double frame_pose[16], const double R[9], const double t[3], double rigid_inv[16])
{
    double inv[16];
    if (!vo_invert_rigid4(R, t, inv)) return VO_E_INVALID;
    if (rigid_inv) memcpy(rigid_inv, inv, sizeof(inv));
    return vo_integrate_rigid(frame_pose, t, inv);
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

__global__ void k_pose_step(int n, double* frame_pose, const double* __restrict__ R, const double* __restrict__ t, int* rc)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double pose[16];
    for (int k = 0; k < 16; k++) pose[k] = frame_pose[16 * (size_t)i + k];
    const int r = vo_pose_step_dev(pose, R + 9 * (size_t)i, t + 3 * (size_t)i);
    for (int k = 0; k < 16; k++) frame_pose[16 * (size_t)i + k] = pose[k];
    rc[i] = r;
}

extern "C" int vo_pose_step_device(vo_ctx* ctx, int n, double* frame_pose, const double* R, const double* t, int* rc)
{
    if (!ctx) return VO_E_INVALID;
    if (n < 0 || (n > 0 && (!frame_pose || !R || !t))) { vo_set_error(ctx, "vo_pose_step_device: bad argument"); return VO_E_INVALID; }
    if (n == 0) return VO_OK;
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const size_t o_R = 16 * (size_t)n * sizeof(double), o_t = o_R + 9 * (size_t)n * sizeof(double);
    const size_t o_rc = o_t + 3 * (size_t)n * sizeof(double), bytes = o_rc + (size_t)n * sizeof(int);
    uint8_t* d = nullptr;
    VO_CUDA_CHECK(cudaMalloc(&d, bytes));
    cudaStream_t st = ctx->stream;
    cudaError_t e = cudaMemcpyAsync(d, frame_pose, o_R, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_R, R, o_t - o_R, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_t, t, o_rc - o_t, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        k_pose_step<<<(n + 127) / 128, 128, 0, st>>>(n, (double*)d, (const double*)(d + o_R), (const double*)(d + o_t), (int*)(d + o_rc));
        ctx->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(frame_pose, d, o_R, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && rc) e = cudaMemcpyAsync(rc, d + o_rc, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    VO_CUDA_CHECK(e);
    return VO_OK;
}
