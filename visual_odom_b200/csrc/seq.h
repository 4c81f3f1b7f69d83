// seq.h -- launch interface of the sequence-mode glue kernels (seq.cu)
#pragma once
#include "common.cuh"
#include "pnp.h"
#include "ess.h"
#include "../../include/vo_b200.h"
#define SEQ_STARTED 2         // vo_ctx::seq_live: the slot's sequence started in this submission (stages skip it)

// The pointers are those of sequence 0; one launch covers n_seq sequences (blockIdx.y = q) and finds sequence q's part of
// each array `stride` elements further on: corner_cap (corners), feat_cap (feat_pts, feat_ages), 2 (cnt), bucket_cap
// (bucket), out_cap (out_pts, out_ages, valid_l1, ages_out), 3 (tprev, tprev_cur), 1 (everything else).
struct SeqArgs {
    // append
    const float2* corners; const int* n_det; int corner_cap;
    float2* feat_pts; int* feat_ages; int* cnt /* [2]: points, ages */; int feat_cap;
    // each sequence's parameter entry (stride 1): the refill threshold (append), and the bucketing's bucket_size = rows /
    // bucket_rows_divisor, features_per_bucket slots per cell, ages >= bucket_age_threshold refused
    const UnitParams* par;
    // bucketing: bucket: last[nb] | first[nb][features_per_bucket] scratch
    int rows, cols; int* bucket; size_t bucket_cap;
    // images of several sizes: sequence q's rows / cols (and so its bucket_size) are those of geo[q * geo_stride]
    const PlaneGeom* geo; int geo_stride;
    float2* out_pts; int* out_ages; int* out_n; int out_cap;
    // update
    const float2* valid_l1; const int* n5; const int* ages_out; const int* n3;
    vo_unit_result_dev* res; double* tprev /* the NEXT frame's t_prev slot */; const double* tprev_cur /* this frame's */;
    int* err; int* err_out /* per-frame copy of the sticky error bits, read back with the record */;
    // 0 once the sequence is retired: its block writes no features (out_n = 0) and leaves its state and translation alone
    const int* live;
};

int vo_launch_seq_append(const SeqArgs& a, int n_seq, cudaStream_t s);
int vo_launch_seq_bucket(const SeqArgs& a, int n_seq, cudaStream_t s);
int vo_launch_seq_carry(const SeqArgs& a, int n_seq, cudaStream_t s);
int vo_launch_seq_finish(const SeqArgs& a, int n_seq, cudaStream_t s);
// mono_rotation = true: each live sequence's record R becomes recoverPose's rotation (I where the branch aborted);
// everything else in the record stays the PnP's.  ess: sequence 0's result, sequence q's ess_stride bytes further on.
int vo_launch_seq_mono(const SeqArgs& a, const EssResult* ess, size_t ess_stride, int n_seq, cudaStream_t s);

// vo_mseq_wait_device: the oldest submission's results (buffer units u0 .. u0 + n_seq - 1) into caller device buffers.
// mode[q]: 1 the sequence ran in that submission, 0 retired or empty, SEQ_STARTED started by it.  Sources are
// sequence 0's (the unit u0) with the strides of SeqArgs (cap for the point lists, ess_stride bytes for ess / ess_mask);
// every destination may be NULL.
struct CollectArgs {
    const vo_unit_result_dev* res; const int* err; int cap;
    const float2* valid4; size_t plane_stride;          // the four lists of unit u0: valid4 + k * plane_stride
    const float3* X; const int* inliers;
    const EssResult* ess; const uint8_t* ess_mask; size_t ess_stride;   // mono runs only (else NULL)
    double* pose;                                       // [n_seq][16] device frame_pose, integrated here
    int* status; vo_unit_result_dev* records; double* pose_out; int pts_cap;
    float2* pts4; float3* points3d; int* inliers_out; vo_mono_result* mono; uint8_t* mask_out;
    unsigned char mode[VO_MSEQ_MAX];
};
int vo_launch_seq_collect(const CollectArgs& a, int n_seq, cudaStream_t s);
