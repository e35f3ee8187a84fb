// GroupNorm kernels of the fused plan that are not convolutions: the seams of the fused data-gradient chain (stand-alone version
// of the fused epilogue, for the layers that stay on the unfused kernels), the finish of the fixed-point (d gamma, d beta)
// accumulators, and the last forward layer (GroupNorm from fixed-point statistics + residual + ReLU, fused with the average pool).
#include "common.cuh"
#include "kernels.h"

namespace dboa {
namespace gnf {

constexpr double FIX = 268435456.0;                      // 2^28 fixed point of the backward sums
constexpr double FIX_FWD = 16777216.0;                   // 2^24 fixed point of the forward statistics
constexpr float GN_EPS = 1e-5f;

struct Prep {                      // GroupNorm whose backward is prepared
    const float* y;                // raw output of layer p [B][H][W][C]
    const float* stats;            // (mean, rstd) [B][4][2]
    const float* gamma;
    unsigned long long* sums;      // [B][4][2]: sum q, sum q x^
    unsigned long long* dgb;       // [C][2]: d gamma, d beta
};
__device__ __forceinline__ long long to_fix(float v) { return __double2ll_rn((double)v * FIX); }

// Stand-alone version of the fused data-gradient epilogue (conv_tc.cu) for the seams with the unfused kernels (after avgpool_bwd; after a stride-2 block):
// dz = dA * (a > 0) -> out; sums / d gamma / d beta of GroupNorm_p.  grid (ceil(HW / rows_per_cta), B), 256 threads: a thread keeps
// its channel vector(s) over the (few) rows of the CTA, all loads of a row group in flight together; the two group sums go
// through a warp butterfly before they touch shared memory (a warp's 32 channel vectors lie in one group for C >= 512; for
// narrower layers the segments are 16 / 8 lanes), so the shared 64-bit adds see at most 8 contenders instead of 256.
__global__ void __launch_bounds__(256) gn_bwd_prep_kernel(const float* __restrict__ dA, const float* __restrict__ mask, float* __restrict__ out,
                                                          Prep p, int HW, int C, int rows_per_cta) {
    __shared__ unsigned long long sacc[8];
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.y, C4 = C >> 2, gw = C >> 2, lane = threadIdx.x & 31;
    const int cvg = C4 >> 2;                                 // channel vectors per group (a power of two >= 4 for the backbone widths)
    const int seg = cvg >= 32 ? 32 : cvg;                    // lanes of a warp that share a group
    if (threadIdx.x < 8) sacc[threadIdx.x] = 0ull;
    __syncthreads();
    const int r_begin = blockIdx.x * rows_per_cta, r_end = min(HW, r_begin + rows_per_cta);
    for (int cv0 = 0; cv0 < C4; cv0 += 256) {                // uniform trip count: every lane takes part in the butterflies
        const int cv = cv0 + threadIdx.x;
        const bool live = cv < C4;
        const int c = live ? cv * 4 : 0, g = c / gw;
        float4 sdg = make_float4(0.f, 0.f, 0.f, 0.f), sdb = sdg;
        float sq = 0.f, sqx = 0.f;
        if (live) {
            const float4 ga = ldg4(p.gamma + c);
            const float mu = __ldg(p.stats + ((size_t)b * 4 + g) * 2), rs = __ldg(p.stats + ((size_t)b * 4 + g) * 2 + 1);
#pragma unroll 4
            for (int r = r_begin; r < r_end; ++r) {
                const size_t e = ((size_t)b * HW + r) * C + c;
                float4 d = __ldcg(reinterpret_cast<const float4*>(dA + e));
                const float4 m = __ldcg(reinterpret_cast<const float4*>(mask + e)), yv = __ldcg(reinterpret_cast<const float4*>(p.y + e));
                d.x = m.x > 0.f ? d.x : 0.f; d.y = m.y > 0.f ? d.y : 0.f; d.z = m.z > 0.f ? d.z : 0.f; d.w = m.w > 0.f ? d.w : 0.f;
                *reinterpret_cast<float4*>(out + e) = d;
                const float x0 = (yv.x - mu) * rs, x1 = (yv.y - mu) * rs, x2 = (yv.z - mu) * rs, x3 = (yv.w - mu) * rs;
                const float q0 = d.x * ga.x, q1 = d.y * ga.y, q2 = d.z * ga.z, q3 = d.w * ga.w;
                sdg.x += d.x * x0; sdg.y += d.y * x1; sdg.z += d.z * x2; sdg.w += d.w * x3;
                sdb.x += d.x; sdb.y += d.y; sdb.z += d.z; sdb.w += d.w;
                sq += (q0 + q1) + (q2 + q3);
                sqx += (q0 * x0 + q1 * x1) + (q2 * x2 + q3 * x3);
            }
        }
        long long a1 = to_fix(sq), a2 = to_fix(sqx);
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1)
            if (o < seg) { a1 += __shfl_xor_sync(0xffffffffu, a1, o); a2 += __shfl_xor_sync(0xffffffffu, a2, o); }
        if (live && (lane & (seg - 1)) == 0) {
            atomicAdd(&sacc[g * 2], (unsigned long long)a1);
            atomicAdd(&sacc[g * 2 + 1], (unsigned long long)a2);
        }
        if (live) {
            const float dgv[4] = {sdg.x, sdg.y, sdg.z, sdg.w}, dbv[4] = {sdb.x, sdb.y, sdb.z, sdb.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                atomicAdd(p.dgb + (size_t)(c + e) * 2, (unsigned long long)to_fix(dgv[e]));
                atomicAdd(p.dgb + (size_t)(c + e) * 2 + 1, (unsigned long long)to_fix(dbv[e]));
            }
        }
    }
    __syncthreads();
    if (threadIdx.x < 8) atomicAdd(p.sums + (size_t)b * 8 + threadIdx.x, sacc[threadIdx.x]);
}

// G[g_off + c] += d gamma, G[b_off + c] += d beta from the fixed-point accumulators of every GroupNorm (one launch per backward)
__global__ void __launch_bounds__(256) gn_dgb_finish_kernel(const GnFinishItem* __restrict__ items, const long long* __restrict__ dgb, float* __restrict__ G) {
    pdl_wait();
    pdl_trigger();
    const GnFinishItem it = items[blockIdx.x];
    const long long* a = dgb + 2 * it.cum_channels;
    for (int c = threadIdx.x; c < it.C; c += 256) {
        const long long vg = a[2 * c], vb = a[2 * c + 1];
        if (vg != 0) G[it.g_off + c] += (float)((double)vg / FIX);
        if (vb != 0) G[it.b_off + c] += (float)((double)vb / FIX);
    }
}

// GroupNorm apply from the fixed-point statistics (+ residual, ReLU) fused with the 7x7 average pool: the last layer of the
// backbone (reference model/hmr.py:57-60 of layer4.2, :156-157).  grid (C / 128, B), 256 threads.
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gn_acc_res_avgpool_kernel(const float* __restrict__ y, const float* __restrict__ res, const long long* __restrict__ acc,
                                                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                  float* __restrict__ a_out, float* __restrict__ stats_out, float* __restrict__ out, int HW,
                                                                  int C, int ld, int ncopy, size_t copy_stride) {
    __shared__ float4 part[8][32];
    __shared__ float sst[8];
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < 4) {
        const long long* a = acc + ((size_t)b * 4 + threadIdx.x) * 2;
        const double N = (double)HW * (C >> 2);
        const double s1 = (double)__ldcg(a) / FIX_FWD, s2 = (double)__ldcg(a + 1) / FIX_FWD;
        const double mu = s1 / N, var = fmax(s2 / N - mu * mu, 0.0);
        sst[threadIdx.x] = (float)mu;
        sst[4 + threadIdx.x] = 1.0f / sqrtf((float)var + GN_EPS);
    }
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < 8 && stats_out != nullptr) stats_out[(b * 4 + (threadIdx.x & 3)) * 2 + (threadIdx.x >> 2)] = sst[threadIdx.x];
    const int c = blockIdx.x * 128 + lane * 4, g = c / (C >> 2);
    const float mu = sst[g], rs = sst[4 + g];
    const float4 ga = ldg4(gamma + c), be = ldg4(beta + c);
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = warp; p < HW; p += 8) {
        const size_t off = ((size_t)b * HW + p) * C + c;
        const float4 v = ldg4(y + off), r = ldg4(res + off);
        float4 o;
        o.x = (v.x - mu) * (rs * ga.x) + be.x; o.y = (v.y - mu) * (rs * ga.y) + be.y;
        o.z = (v.z - mu) * (rs * ga.z) + be.z; o.w = (v.w - mu) * (rs * ga.w) + be.w;
        o.x = fmaxf(o.x + r.x, 0.f); o.y = fmaxf(o.y + r.y, 0.f); o.z = fmaxf(o.z + r.z, 0.f); o.w = fmaxf(o.w + r.w, 0.f);
        *reinterpret_cast<float4*>(a_out + off) = o;
        s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
    }
    part[warp][lane] = s;
    __syncthreads();
    if (warp == 0) {
        float4 t = part[0][lane];
        for (int w = 1; w < 8; ++w) { const float4 q = part[w][lane]; t.x += q.x; t.y += q.y; t.z += q.z; t.w += q.w; }
        const float hw = (float)HW;
        t.x /= hw; t.y /= hw; t.z /= hw; t.w /= hw;
        for (int k = 0; k < ncopy; ++k) *reinterpret_cast<float4*>(out + k * copy_stride + (size_t)b * ld + c) = t;
    }
}

}  // namespace gnf

int gn_bwd_prep(const float* dA, const float* mask, float* out, const DgradPrep& p, int B, int HW, int C, cudaStream_t st) {
    if (C % 4 != 0 || C / 4 > 512) return DBOA_ERR_SHAPE;
    gnf::Prep pp;
    pp.y = p.y; pp.stats = p.stats; pp.gamma = p.gamma; pp.sums = reinterpret_cast<unsigned long long*>(p.sums); pp.dgb = reinterpret_cast<unsigned long long*>(p.dgb);
    // enough CTAs to cover the GPU with SHORT row loops (the kernel is a latency chain: a row is one memory round trip)
    int rows_per = 1;
    while (rows_per < 8 && ceil_div(HW, rows_per * 2) * B >= num_sms()) rows_per *= 2;
    return launch_ex(gnf::gn_bwd_prep_kernel, dim3(ceil_div(HW, rows_per), B), dim3(256), 0, st, dim3(1, 1, 1), true, dA, mask, out, pp, HW, C, rows_per);
}

int gn_dgb_finish(const GnFinishItem* items_dev, int n_items, const float* dgb, float* G, cudaStream_t st) {
    return launch_ex(gnf::gn_dgb_finish_kernel, dim3(n_items), dim3(256), 0, st, dim3(1, 1, 1), true, items_dev, reinterpret_cast<const long long*>(dgb), G);
}

int gn_acc_res_avgpool(const float* y, const float* res, const float* acc, const float* gamma, const float* beta, float* a_out, float* stats_out,
                       float* out, int B, int HW, int C, int ld, int ncopy, size_t copy_stride, cudaStream_t st) {
    if (C % 128 != 0 || ld % 4 != 0 || copy_stride % 4 != 0) return DBOA_ERR_SHAPE;
    return launch_ex(gnf::gn_acc_res_avgpool_kernel, dim3(C / 128, B), dim3(256), 0, st, dim3(1, 1, 1), true, y, res, reinterpret_cast<const long long*>(acc), gamma,
                     beta, a_out, stats_out, out, HW, C, ld, ncopy, copy_stride);
}

}  // namespace dboa
