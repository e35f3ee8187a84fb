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
int adam_ema(float* p, const float* g, float* m, float* v, float* teacher, size_t n, float lr, float beta1, float beta2, float eps, int step,
             float alpha, float gscale, cudaStream_t st);
int ema_update(float* teacher, const float* p, size_t n, float alpha, cudaStream_t st);
// out[i] = cos(a_i, b_i) (NULL to skip); terms[i] = (a.b, |a|^2, |b|^2) in double (NULL to skip): the data-parallel feature test all-reduces them.
// Per video g whose bit is set in `active`: out[g][i], terms[g][i], each from video g's parts alone; the rows of other videos
// are not written.  cp.n / groups / active are checked by the caller (n: total lengths, divisible by groups).
int cosine_pairs(const CosinePairs& cp, float* partial, size_t partial_floats, float* out, double* terms, float eps, cudaStream_t st,
                 int groups = 1, unsigned long long active = 1ULL);
long long cosine_partial_floats(const long long* n, int npairs, int groups = 1);
int retrieval_nearest(const float* feat, const float* centers, int K, int D, int* best, float* dists, cudaStream_t st);

}  // namespace dboa
