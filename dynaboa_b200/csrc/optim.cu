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

// float4 i of one Adam (+ EMA) step, shared by the sweeps below, which differ only in where they read their scalars from
__device__ __forceinline__ void adam_ema_at(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                            float* __restrict__ teacher, size_t i, float w1, float b2, float one_m_b2, float bc2_sqrt,
                                            float eps, float neg_step, float alpha, float one_m_alpha, float gscale) {
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
// the scalars from a device block (adam_scalars' order): a replayed CUDA graph reads the bias correction of the current step
__global__ void __launch_bounds__(256) adam_ema_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                           float* __restrict__ v, float* __restrict__ teacher, size_t n4,
                                                           const float* __restrict__ s) {
    const float w1 = s[0], b2 = s[1], one_m_b2 = s[2], bc2_sqrt = s[3], eps = s[4], neg_step = s[5], alpha = s[6], one_m_alpha = s[7],
                gscale = s[8];
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (size_t)gridDim.x * 256)
        adam_ema_at(p, g, m, v, teacher, i, w1, b2, one_m_b2, bc2_sqrt, eps, neg_step, alpha, one_m_alpha, gscale);
}

// ---------------------------------------------------------------------------------------------
// per-video sweeps: video g owns the float4s [g n4, (g + 1) n4) of every arena and has its own scalars, which travel in the
// launch parameters (no device table); a one-arena call is one video.  The grid strides over the active videos' float4s as
// over one arena of nact * n4 float4s, with the one-arena sweep's grid: step j of the walk is float4 j % n4 of the (j / n4)-th
// active video (t.video), the pair advanced by subtraction rather than division.
// ---------------------------------------------------------------------------------------------
struct VideoSweep {
    float s[MAX_VIDEOS][ADAM_SCALARS];      // SGD: s[g][0] = -lr of video g; Adam: dboa_adam_scalars' row of video g
    unsigned char video[MAX_VIDEOS];
};

// the active videos into t.video; returns their number
static int active_videos(VideoSweep& t, int groups, unsigned long long active) {
    int nact = 0;
    for (int g = 0; g < groups; ++g)
        if ((active >> g) & 1ULL) t.video[nact++] = (unsigned char)g;
    return nact;
}

// calls at(video, float4 index in the stack) for every float4 of the walk this thread takes
template <class At>
__device__ __forceinline__ void video_walk(size_t n4, int nact, const VideoSweep& t, const At& at) {
    const size_t total = n4 * nact, stride = (size_t)gridDim.x * 256;
    size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    int k = (int)(i / n4);
    size_t off = i - (size_t)k * n4;
    for (; i < total; i += stride) {
        const int v = t.video[k];
        at(v, (size_t)v * n4 + off);
        off += stride;
        while (off >= n4) { off -= n4; ++k; }
    }
}

__global__ void __launch_bounds__(256) sgd_update_groups_kernel(const float* __restrict__ p, const float* __restrict__ g, float* __restrict__ out,
                                                                size_t n4, int nact, const VideoSweep t) {
    video_walk(n4, nact, t, [&](int v, size_t i) {
        const float neg_lr = t.s[v][0];
        float4 a = reinterpret_cast<const float4*>(p)[i], b = reinterpret_cast<const float4*>(g)[i], o;
        o.x = __fadd_rn(a.x, __fmul_rn(neg_lr, b.x)); o.y = __fadd_rn(a.y, __fmul_rn(neg_lr, b.y));
        o.z = __fadd_rn(a.z, __fmul_rn(neg_lr, b.z)); o.w = __fadd_rn(a.w, __fmul_rn(neg_lr, b.w));
        reinterpret_cast<float4*>(out)[i] = o;
    });
}
int sgd_update(const float* p, const float* g, float* out, float lr, size_t n, cudaStream_t st) {
    if (n % 4) return DBOA_ERR_SHAPE;
    return sgd_update_groups(p, g, out, &lr, n, 1, 1ULL, st);
}
int sgd_update_groups(const float* p, const float* g, float* out, const float* lr, size_t n, int groups, unsigned long long active,
                      cudaStream_t st) {
    VideoSweep t;
    for (int v = 0; v < groups; ++v)
        if ((active >> v) & 1ULL) t.s[v][0] = -lr[v];
    const int nact = active_videos(t, groups, active);
    sgd_update_groups_kernel<<<sweep_grid(n / 4 * nact), 256, 0, st>>>(p, g, out, n / 4, nact, t);
    return check_launch();
}

__global__ void __launch_bounds__(256) adam_ema_groups_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                              float* __restrict__ v, float* __restrict__ teacher, size_t n4, int nact,
                                                              const VideoSweep t) {
    video_walk(n4, nact, t, [&](int k, size_t i) {
        adam_ema_at(p, g, m, v, teacher, i, t.s[k][0], t.s[k][1], t.s[k][2], t.s[k][3], t.s[k][4], t.s[k][5], t.s[k][6], t.s[k][7], t.s[k][8]);
    });
}
void adam_scalars(double lr, double beta1, double beta2, double eps, int step, double alpha, float gscale, float out[ADAM_SCALARS]) {
    // torch.optim.Adam (single-tensor path) derives these from the hyperparameters in Python doubles, then casts each
    // scalar once to fp32: so does this, from the caller's doubles (1 - beta2 of a float-rounded beta2 is off by ulps)
    const double bc1 = 1.0 - pow(beta1, step), bc2 = 1.0 - pow(beta2, step);
    out[0] = (float)(1.0 - beta1); out[1] = (float)beta2; out[2] = (float)(1.0 - beta2); out[3] = (float)sqrt(bc2); out[4] = (float)eps;
    out[5] = (float)(-(lr / bc1)); out[6] = (float)alpha; out[7] = (float)(1.0 - alpha); out[8] = gscale;
}
int adam_ema(float* p, const float* g, float* m, float* v, float* teacher, size_t n, double lr, double beta1, double beta2, double eps,
             int step, double alpha, float gscale, cudaStream_t st) {
    if (n % 4 || step < 1) return DBOA_ERR_ARG;
    float s[ADAM_SCALARS];
    adam_scalars(lr, beta1, beta2, eps, step, alpha, gscale, s);
    return adam_ema_groups(p, g, m, v, teacher, n, s, 1, 1ULL, st);
}
int adam_ema_dev(float* p, const float* g, float* m, float* v, float* teacher, size_t n, const float* scalars, cudaStream_t st) {
    if (n % 4) return DBOA_ERR_ARG;
    adam_ema_dev_kernel<<<sweep_grid(n / 4), 256, 0, st>>>(p, g, m, v, teacher, n / 4, scalars);
    return check_launch();
}
int adam_ema_groups(float* p, const float* g, float* m, float* v, float* teacher, size_t n, const float* scalars, int groups,
                    unsigned long long active, cudaStream_t st) {
    VideoSweep t;
    for (int k = 0; k < groups; ++k)
        if ((active >> k) & 1ULL)
            for (int i = 0; i < ADAM_SCALARS; ++i) t.s[k][i] = scalars[k * ADAM_SCALARS + i];
    const int nact = active_videos(t, groups, active);
    adam_ema_groups_kernel<<<sweep_grid(n / 4 * nact), 256, 0, st>>>(p, g, m, v, teacher, n / 4, nact, t);
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
int ema_update(float* teacher, const float* p, size_t n, double alpha, cudaStream_t st) {
    if (n % 4) return DBOA_ERR_SHAPE;
    ema_kernel<<<sweep_grid(n / 4), 256, 0, st>>>(teacher, p, n / 4, (float)alpha, (float)(1.0 - alpha));
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
