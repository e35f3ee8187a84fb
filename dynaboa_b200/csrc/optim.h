#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace dboa {

// npairs tensor pairs a[i], b[i] of n[i] floats.  cosine_pairs fills the rest for the kernels: n[i] becomes the length of one
// video's part (video g's part of pair i starts at a[i] + g * n[i]), blk_off counts the COS_CHUNK blocks of one video, and
// video[k] is the k-th active video.
struct CosinePairs {
    const float* a[16];
    const float* b[16];
    long long n[16];
    int blk_off[17];
    int npairs;
    unsigned char video[64];
};

int sgd_update(const float* p, const float* g, float* out, float lr, size_t n, cudaStream_t st);
int adam_ema(float* p, const float* g, float* m, float* v, float* teacher, size_t n, double lr, double beta1, double beta2, double eps,
             int step, double alpha, float gscale, cudaStream_t st);
// the fp32 scalars of one Adam (+ EMA) sweep, in this order: 1 - beta1, beta2, 1 - beta2, sqrt(bias correction 2), eps,
// -(lr / bias correction 1), alpha, 1 - alpha, gscale
constexpr int ADAM_SCALARS = 9;
void adam_scalars(double lr, double beta1, double beta2, double eps, int step, double alpha, float gscale, float out[ADAM_SCALARS]);
// adam_ema with the scalars read from the device block `scalars` (ADAM_SCALARS floats) when the kernel runs
int adam_ema_dev(float* p, const float* g, float* m, float* v, float* teacher, size_t n, const float* scalars, cudaStream_t st);
// Per-video sweeps over `groups` (1..64) arenas of n floats each, only the videos whose bit is set in `active` (others: not read,
// not written).  lr: host (groups,) array, video g's learning rate; scalars: host (groups, ADAM_SCALARS) array, video g's row of
// adam_scalars.  sgd_update and adam_ema are these sweeps over one video; video g's floats are bit-identical to adam_ema_dev over
// its arenas with its scalars.  The caller checks the arguments (n % 4 == 0, groups, active).
int sgd_update_groups(const float* p, const float* g, float* out, const float* lr, size_t n, int groups, unsigned long long active,
                      cudaStream_t st);
int adam_ema_groups(float* p, const float* g, float* m, float* v, float* teacher, size_t n, const float* scalars, int groups,
                    unsigned long long active, cudaStream_t st);
int ema_update(float* teacher, const float* p, size_t n, double alpha, cudaStream_t st);
// out[i] = cos(a_i, b_i) (NULL to skip); terms[i] = (a.b, |a|^2, |b|^2) in double (NULL to skip): the data-parallel feature test all-reduces them.
// Per video g whose bit is set in `active`: out[g][i], terms[g][i], each from video g's parts alone; the rows of other videos
// are not written.  cp.n / groups / active are checked by the caller (n: total lengths, divisible by groups).
int cosine_pairs(const CosinePairs& cp, float* partial, size_t partial_floats, float* out, double* terms, float eps, cudaStream_t st,
                 int groups = 1, unsigned long long active = 1ULL);
long long cosine_partial_floats(const long long* n, int npairs, int groups = 1);
int retrieval_nearest(const float* feat, const float* centers, int K, int D, int* best, float* dists, cudaStream_t st);

}  // namespace dboa
