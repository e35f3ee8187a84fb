// Internal argument block of the multi-term loss head (mirrors dboa_loss_args of the public header).
#pragma once
#include <cuda_runtime.h>
#include "../../include/dynaboa_b200.h"

namespace dboa {

typedef dboa_loss_args LossArgs;

int project_fwd_launch(const float* cam, const float* j3d, float* p2d, int B, int NJ, cudaStream_t st);
int project_bwd_launch(const float* cam, const float* j3d, const float* dp2d, float* dj3d, float* dcam, int B, int NJ, int acc_j, int acc_c,
                       cudaStream_t st);
int pose_prior_launch(const float* rot, const float* means, const float* prec, const float* neg_log_w, float* prior_b, float* drot,
                      float scale, int B, cudaStream_t st);
int gmm_prior_launch(const float* pose69, const float* means, const float* prec, const float* neg_log_w, float* prior_b, float* dpose,
                     float scale, int B, cudaStream_t st);
int loss_multi_launch(const LossArgs& a, cudaStream_t st);
int loss_motion_launch(const float* pa, const float* ph, const float* ka, const float* kh, float w, float* term, float* dpa, float* dph,
                       int B, int acc_a, int first, int count, cudaStream_t st, int groups = 1, unsigned long long active = ~0ULL);

}  // namespace dboa
