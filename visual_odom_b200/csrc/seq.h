// seq.h -- launch interface of the sequence-mode glue kernels (seq.cu)
#pragma once
#include "common.cuh"
#include "pnp.h"
#include "ess.h"

struct SeqArgs {
    // append
    const float2* corners; const int* n_det; int corner_cap;
    float2* feat_pts; int* feat_ages; int* cnt /* [2]: points, ages */; int feat_cap; int refill_below;
    // bucketing
    int rows, cols, bucket_size; int* bucket; int bucket_cap;
    float2* out_pts; int* out_ages; int* out_n; int out_cap;
    // update
    const float2* valid_l1; const int* n5; const int* ages_out; const int* n3;
    vo_unit_result_dev* res; double* tprev /* the NEXT frame's t_prev slot */;
    int* err; int* err_out /* per-frame copy of the sticky error bits, read back with the record */;
};

int vo_launch_seq_append(const SeqArgs& a, cudaStream_t s);
int vo_launch_seq_bucket(const SeqArgs& a, cudaStream_t s);
int vo_launch_seq_carry(const SeqArgs& a, cudaStream_t s);
int vo_launch_seq_finish(const SeqArgs& a, cudaStream_t s);
// mono_rotation = true: the record's R becomes recoverPose's rotation (I where the branch aborted); everything else in
// the record stays the PnP's
int vo_launch_seq_mono(vo_unit_result_dev* res, const EssResult* ess, cudaStream_t s);
