// Whole-model elementwise sweeps over the flat parameter arena, the 15-feature cosine test and
// exemplar-cluster retrieval.
//
// Replaces: learn2learn maml_update (p' = p + (-lr * g), reference dynaboa_benchmark.py:140;
// SURVEY.md K12), torch.optim.Adam.step (reference base_adaptor.py:126, K13), update_teacher
// (base_adaptor.py:193-201, K14) -- 169 x 2 tiny launches each in the reference, one launch here --
// cal_feature_diff (base_adaptor.py:211-219, K15: 15 cosines + 15 host syncs -> one launch, one sync)
// and retrieval's nearest-centre search (base_adaptor.py:82-84, K16).
#include "common.cuh"
#include "kernels.h"
#include "optim.h"

namespace dboa {

static inline int sweep_grid(size_t n4) {
    size_t blocks = (n4 + 255) / 256;
    size_t cap = (size_t)num_sms() * 16;
    return (int)(blocks < cap ? (blocks ? blocks : 1) : cap);
}

__global__ void __launch_bounds__(256) sgd_update_kernel(const float* __restrict__ p, const float* __restrict__ g, float* __restrict__ out,
                                                         float neg_lr, size_t n4) {
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (size_t)gridDim.x * 256) {
        float4 a = reinterpret_cast<const float4*>(p)[i], b = reinterpret_cast<const float4*>(g)[i], o;
        o.x = __fadd_rn(a.x, __fmul_rn(neg_lr, b.x)); o.y = __fadd_rn(a.y, __fmul_rn(neg_lr, b.y));
        o.z = __fadd_rn(a.z, __fmul_rn(neg_lr, b.z)); o.w = __fadd_rn(a.w, __fmul_rn(neg_lr, b.w));
        reinterpret_cast<float4*>(out)[i] = o;
    }
}
int sgd_update(const float* p, const float* g, float* out, float lr, size_t n, cudaStream_t st) {
    if (n % 4) return DBOA_ERR_SHAPE;
    sgd_update_kernel<<<sweep_grid(n / 4), 256, 0, st>>>(p, g, out, -lr, n / 4);
    return check_launch();
}

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, float w1, float b2, float one_m_b2, float bc2_sqrt,
                                         float eps, float neg_step) {
    // exp_avg.lerp_(grad, 1 - beta1): ATen evaluates  w < 0.5 ? a + w (b - a) : b - (b - a)(1 - w)
    const float diff = __fsub_rn(g, m);
    m = (w1 < 0.5f) ? __fadd_rn(m, __fmul_rn(w1, diff)) : __fsub_rn(g, __fmul_rn(diff, __fsub_rn(1.0f, w1)));
    // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2)
    v = __fadd_rn(__fmul_rn(v, b2), __fmul_rn(__fmul_rn(one_m_b2, g), g));
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
    p = __fadd_rn(p, __fmul_rn(neg_step, __fdiv_rn(m, denom)));
}

__global__ void __launch_bounds__(256) adam_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                       float* __restrict__ v, float* __restrict__ teacher, size_t n4, float w1, float b2,
                                                       float one_m_b2, float bc2_sqrt, float eps, float neg_step, float alpha,
                                                       float one_m_alpha, float gscale) {
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (size_t)gridDim.x * 256) {
        float4 pp = reinterpret_cast<float4*>(p)[i], gg = reinterpret_cast<const float4*>(g)[i];
        float4 mm = reinterpret_cast<float4*>(m)[i], vv = reinterpret_cast<float4*>(v)[i];
        // data-parallel mean of the all-reduced (summed) gradient: g / R folded into this sweep (1.0f is exact: single-GPU results unchanged)
        gg.x = __fmul_rn(gg.x, gscale); gg.y = __fmul_rn(gg.y, gscale); gg.z = __fmul_rn(gg.z, gscale); gg.w = __fmul_rn(gg.w, gscale);
        adam_one(pp.x, gg.x, mm.x, vv.x, w1, b2, one_m_b2, bc2_sqrt, eps, neg_step);
        adam_one(pp.y, gg.y, mm.y, vv.y, w1, b2, one_m_b2, bc2_sqrt, eps, neg_step);
        adam_one(pp.z, gg.z, mm.z, vv.z, w1, b2, one_m_b2, bc2_sqrt, eps, neg_step);
        adam_one(pp.w, gg.w, mm.w, vv.w, w1, b2, one_m_b2, bc2_sqrt, eps, neg_step);
        reinterpret_cast<float4*>(p)[i] = pp; reinterpret_cast<float4*>(m)[i] = mm; reinterpret_cast<float4*>(v)[i] = vv;
        if (teacher != nullptr) {
            float4 tt = reinterpret_cast<float4*>(teacher)[i];
            tt.x = __fadd_rn(__fmul_rn(tt.x, alpha), __fmul_rn(one_m_alpha, pp.x));
            tt.y = __fadd_rn(__fmul_rn(tt.y, alpha), __fmul_rn(one_m_alpha, pp.y));
            tt.z = __fadd_rn(__fmul_rn(tt.z, alpha), __fmul_rn(one_m_alpha, pp.z));
            tt.w = __fadd_rn(__fmul_rn(tt.w, alpha), __fmul_rn(one_m_alpha, pp.w));
            reinterpret_cast<float4*>(teacher)[i] = tt;
        }
    }
}
int adam_ema(float* p, const float* g, float* m, float* v, float* teacher, size_t n, float lr, float beta1, float beta2, float eps,
             int step, float alpha, float gscale, cudaStream_t st) {
    if (n % 4 || step < 1) return DBOA_ERR_ARG;
    // torch.optim.Adam (single-tensor path) computes these in Python doubles, then casts the scalars
    double bc1 = 1.0 - pow((double)beta1, step), bc2 = 1.0 - pow((double)beta2, step);
    float neg_step = (float)(-((double)lr / bc1)), bc2_sqrt = (float)sqrt(bc2);
    adam_ema_kernel<<<sweep_grid(n / 4), 256, 0, st>>>(p, g, m, v, teacher, n / 4, (float)(1.0 - (double)beta1), beta2,
                                                       (float)(1.0 - (double)beta2), bc2_sqrt, eps, neg_step, alpha,
                                                       (float)(1.0 - (double)alpha), gscale);
    return check_launch();
}

__global__ void __launch_bounds__(256) ema_kernel(float* __restrict__ t, const float* __restrict__ p, size_t n4, float alpha, float oma) {
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (size_t)gridDim.x * 256) {
        float4 tt = reinterpret_cast<float4*>(t)[i], pp = reinterpret_cast<const float4*>(p)[i];
        tt.x = __fadd_rn(__fmul_rn(tt.x, alpha), __fmul_rn(oma, pp.x)); tt.y = __fadd_rn(__fmul_rn(tt.y, alpha), __fmul_rn(oma, pp.y));
        tt.z = __fadd_rn(__fmul_rn(tt.z, alpha), __fmul_rn(oma, pp.z)); tt.w = __fadd_rn(__fmul_rn(tt.w, alpha), __fmul_rn(oma, pp.w));
        reinterpret_cast<float4*>(t)[i] = tt;
    }
}
int ema_update(float* teacher, const float* p, size_t n, float alpha, cudaStream_t st) {
    if (n % 4) return DBOA_ERR_SHAPE;
    ema_kernel<<<sweep_grid(n / 4), 256, 0, st>>>(teacher, p, n / 4, alpha, (float)(1.0 - (double)alpha));
    return check_launch();
}

// ---------------------------------------------------------------------------------------------
// cosine similarity of up to 16 tensor pairs in two launches (partials, then a fixed-order finish), for each of up to 64
// videos on its own part of every pair.  The grids cover the active videos only (blockIdx.y / blockIdx.x of the finish is the
// k-th active video), so every CTA waits on its predecessor.  A video's blocks chunk its part from the part's first float and
// its partials sit at the offsets a one-video call would use, shifted by g * blk_off[npairs]: its sums are those of the call
// on its parts alone, bit for bit.
// ---------------------------------------------------------------------------------------------
constexpr int COS_CHUNK = 256 * 16;

__global__ void __launch_bounds__(256) cosine_partial_kernel(CosinePairs cp, float* __restrict__ partial) {
    pdl_wait();
    pdl_trigger();
    __shared__ float red[32];
    const int g = cp.video[blockIdx.y];
    int pair = 0;
    while (pair + 1 < cp.npairs && (int)blockIdx.x >= cp.blk_off[pair + 1]) ++pair;
    const long long beg = (long long)(blockIdx.x - cp.blk_off[pair]) * COS_CHUNK;
    const long long end = beg + COS_CHUNK < cp.n[pair] ? beg + COS_CHUNK : cp.n[pair];
    const float* a = cp.a[pair] + g * cp.n[pair];
    const float* b = cp.b[pair] + g * cp.n[pair];
    float ab = 0.f, aa = 0.f, bb = 0.f;
    for (long long i = beg + threadIdx.x; i < end; i += 256) {
        float x = a[i], y = b[i];
        ab = fmaf(x, y, ab); aa = fmaf(x, x, aa); bb = fmaf(y, y, bb);
    }
    ab = block_sum(ab, red); aa = block_sum(aa, red); bb = block_sum(bb, red);
    if (threadIdx.x == 0) {
        float* p = partial + ((size_t)g * cp.blk_off[cp.npairs] + blockIdx.x) * 3;
        p[0] = ab; p[1] = aa; p[2] = bb;
    }
}
__global__ void cosine_finish_kernel(CosinePairs cp, const float* __restrict__ partial, float* __restrict__ out, double* __restrict__ terms,
                                     float eps) {
    pdl_wait();
    pdl_trigger();
    const int g = cp.video[blockIdx.x];
    int pair = threadIdx.x;
    if (pair >= cp.npairs) return;
    partial += (size_t)g * cp.blk_off[cp.npairs] * 3;
    double ab = 0, aa = 0, bb = 0;
    for (int k = cp.blk_off[pair]; k < cp.blk_off[pair + 1]; ++k) { ab += partial[k * 3]; aa += partial[k * 3 + 1]; bb += partial[k * 3 + 2]; }
    const int row = g * cp.npairs + pair;
    if (terms != nullptr) { terms[row * 3] = ab; terms[row * 3 + 1] = aa; terms[row * 3 + 2] = bb; }
    double na = sqrt(aa), nb = sqrt(bb);
    na = na < eps ? eps : na; nb = nb < eps ? eps : nb;
    if (out != nullptr) out[row] = (float)(ab / (na * nb));
}
long long cosine_partial_floats(const long long* n, int npairs, int groups) {
    long long blocks = 0;
    for (int i = 0; i < npairs; ++i) blocks += ceil_div(n[i] / groups, COS_CHUNK);
    return 3 * blocks * groups;
}
int cosine_pairs(const CosinePairs& cp_in, float* partial, size_t partial_floats, float* out, double* terms, float eps, cudaStream_t st,
                 int groups, unsigned long long active) {
    CosinePairs cp = cp_in;
    if (cp.npairs < 1 || cp.npairs > 16) return DBOA_ERR_ARG;
    int nact = 0;
    for (int g = 0; g < groups; ++g)
        if ((active >> g) & 1ULL) cp.video[nact++] = (unsigned char)g;
    cp.blk_off[0] = 0;
    for (int i = 0; i < cp.npairs; ++i) {
        cp.n[i] /= groups;
        cp.blk_off[i + 1] = cp.blk_off[i] + ceil_div(cp.n[i], COS_CHUNK);
    }
    const int nblk = cp.blk_off[cp.npairs];
    if ((size_t)nblk * 3 * groups > partial_floats) return DBOA_ERR_ARG;
    DBOA_TRY(launch_ex(cosine_partial_kernel, dim3(nblk, nact), dim3(256), 0, st, dim3(1, 1, 1), true, cp, partial));
    return launch_ex(cosine_finish_kernel, dim3(nact), dim3(32), 0, st, dim3(1, 1, 1), true, cp, partial, out, terms, eps);
}

// nearest cluster centre by cosine distance: one block, warp per centre (round robin)
__global__ void __launch_bounds__(256) retrieval_kernel(const float* __restrict__ feat, const float* __restrict__ centers, int K, int D,
                                                        int* __restrict__ best, float* __restrict__ dists) {
    pdl_wait();
    pdl_trigger();
    __shared__ float sd[64];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float ff = 0.f;
    for (int i = lane; i < D; i += 32) ff = fmaf(feat[i], feat[i], ff);
    ff = warp_sum(ff);
    for (int k = w; k < K; k += 8) {
        float fc = 0.f, cc = 0.f;
        for (int i = lane; i < D; i += 32) { float c = centers[(size_t)k * D + i]; fc = fmaf(feat[i], c, fc); cc = fmaf(c, c, cc); }
        fc = warp_sum(fc); cc = warp_sum(cc);
        if (lane == 0) sd[k] = 1.0f - fc / (fmaxf(sqrtf(ff), 1e-8f) * fmaxf(sqrtf(cc), 1e-8f));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int b = 0;
        for (int k = 0; k < K; ++k) { dists[k] = sd[k]; if (sd[k] < sd[b]) b = k; }
        best[0] = b;
    }
}
int retrieval_nearest(const float* feat, const float* centers, int K, int D, int* best, float* dists, cudaStream_t st) {
    if (K < 1 || K > 64) return DBOA_ERR_SHAPE;
    return launch_ex(retrieval_kernel, dim3(1), dim3(256), 0, st, dim3(1, 1, 1), true, feat, centers, K, D, best, dists);
}

}  // namespace dboa
