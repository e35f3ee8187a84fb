// GroupNorm(4 groups) forward / backward on NHWC fp32 activations, one launch each.
//
// Replaces the ATen kernels behind reference model/hmr.py:14-18 (gn_helper -> nn.GroupNorm(4, C),
// eps 1e-5, affine) and :36/57-58 (ReLU, residual add) -- SURVEY.md section 2.1 K2/K3.
//
// At batch 1 every layer is a few-microsecond problem: what sets the time is the number of DEPENDENT
// steps (memory round trips, barriers) and the number of instructions each thread issues with few
// warps to hide their latency -- not bytes.  Hence:
//   * one (sample, group) is handled by ONE thread-block cluster of <= 16 CTAs x 1024 threads; every
//     thread owns <= 4 float4 (same channels, rows a fixed stride apart: no integer division, the
//     channels-per-group count is a power of two);
//   * ALL global loads are issued up front into registers (one round trip); every tensor is read once;
//   * the CTAs publish their partial sums in shared memory, barrier.cluster, and every CTA combines
//     all partials through distributed shared memory with a fixed shuffle tree (deterministic);
//   * statistics are (count, mean, M2) per CTA merged with the pairwise formula, robust to large means;
//   * the affine-parameter gradients are reduced per channel inside the CTA (shuffles + one shared
//     pass), across the cluster through DSMEM, and added to dgamma / dbeta directly at batch 1; with
//     several samples the per-sample rows go through global memory and are summed in sample order
//     (deterministic) -- by the last cluster of a group (stand-alone call), or for the whole network by
//     ONE gn_param_finish launch at the end of the backward (`defer`: no fence / ticket per layer).
#include <cooperative_groups.h>

#include "common.cuh"
#include "kernels.h"

namespace cg = cooperative_groups;

namespace dboa {

constexpr int GN_G = 4;
constexpr float GN_EPS = 1e-5f;
constexpr int GN_NT = 1024;                      // threads per CTA
constexpr int GN_V = 4;                          // float4 per thread held in registers
constexpr int GN_MAXCL = 16;                     // CTAs per cluster (non-portable limit)

struct GnPlan { int chunks, rows, lg; };
// chunks CTAs per (sample, group), each `rows` rows of the HW axis; aims at <= 2 float4 per thread
static bool gn_plan(int HW, int C, GnPlan* pl) {
    if (C % 16 != 0) return false;
    const int cg4 = C / GN_G / 4;
    if (cg4 < 1 || cg4 > GN_NT || (cg4 & (cg4 - 1)) != 0) return false;
    int lg = 0;
    while ((1 << lg) < cg4) ++lg;
    const long long nvec = (long long)HW * cg4;
    int chunks = ceil_div(nvec, GN_NT * 2);
    if (chunks > GN_MAXCL) chunks = GN_MAXCL;
    if (chunks < 1) chunks = 1;
    int rows = ceil_div(HW, chunks);
    if ((long long)rows * cg4 > (long long)GN_NT * GN_V) return false;
    chunks = ceil_div(HW, rows);
    pl->chunks = chunks; pl->rows = rows; pl->lg = lg;
    return true;
}

size_t gn_partial_floats(int, int, int) { return 0; }                                // forward needs no global scratch
size_t gn_bwd_partial_floats(int B, int, int C) { return 2 * (size_t)B * C; }        // per-sample dgamma / dbeta rows (B > 1)

static unsigned* g_sync_base = nullptr;
static unsigned* sync_words() {
    if (g_sync_base == nullptr) {
        void* p = nullptr;
        if (cudaMalloc(&p, 64 * sizeof(unsigned)) != cudaSuccess) return nullptr;
        if (cudaMemset(p, 0, 64 * sizeof(unsigned)) != cudaSuccess) return nullptr;
        g_sync_base = static_cast<unsigned*>(p);
    }
    return g_sync_base;
}

// sums of two values over the CTA (fixed tree); valid in every thread.  `red` holds 64 floats and is used once.
__device__ __forceinline__ float2 block_sum2(float a, float b, float* red) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    a = warp_sum(a); b = warp_sum(b);
    if (lane == 0) { red[wid] = a; red[32 + wid] = b; }
    __syncthreads();
    return make_float2(warp_sum(red[lane]), warp_sum(red[32 + lane]));
}

// grid (chunks, 4, B), cluster (chunks, 1, 1)
__global__ void __launch_bounds__(GN_NT, 1) gn_fwd_fused_kernel(const float* __restrict__ y, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, const float* __restrict__ res,
                                                             float* __restrict__ out, float* __restrict__ stats, int HW, int C, int R,
                                                             int lg, int relu) {
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ float red1[64], red2[64];
    __shared__ float part[4];                 // this CTA's (count, mean, M2)
    __shared__ float sm[2];
    pdl_wait();
    pdl_trigger();
    const int chunk = blockIdx.x, g = blockIdx.y, b = blockIdx.z, chunks = gridDim.x;
    const int cg4 = 1 << lg, cgc = cg4 * 4;
    const int r0 = chunk * R, rows = min(R, HW - r0);
    const int cv = threadIdx.x & (cg4 - 1), rt = threadIdx.x >> lg, rstep = GN_NT >> lg;
    const size_t e0 = ((size_t)b * HW + r0 + rt) * C + g * cgc + cv * 4;
    const size_t estep = (size_t)rstep * C;
    const float4 ga = ldg4(gamma + g * cgc + cv * 4), be = ldg4(beta + g * cgc + cv * 4);
    float4 v[GN_V], rr[GN_V];
    bool ok[GN_V];
#pragma unroll
    for (int i = 0; i < GN_V; ++i) {
        ok[i] = rt + i * rstep < rows;
        v[i] = ok[i] ? ldg4(y + e0 + i * estep) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (res != nullptr) rr[i] = ok[i] ? ldg4(res + e0 + i * estep) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < GN_V; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float cnt = (float)(rows * cgc);
    const float cmean = block_sum2(s, 0.f, red1).x / cnt;
    float m2 = 0.f;
#pragma unroll
    for (int i = 0; i < GN_V; ++i) {
        if (ok[i]) {
            float a = v[i].x - cmean, c = v[i].y - cmean, e = v[i].z - cmean, f = v[i].w - cmean;
            m2 += (a * a + c * c) + (e * e + f * f);
        }
    }
    m2 = block_sum2(m2, 0.f, red2).x;
    if (threadIdx.x == 0) { part[0] = cnt; part[1] = cmean; part[2] = m2; }
    cluster.sync();
    if (threadIdx.x < 32) {                                  // merge the chunks' (count, mean, M2): fixed shuffle tree
        const int lane = threadIdx.x;
        float nb = 0.f, mb = 0.f, Mb = 0.f;
        if (lane < chunks) {
            const float* rp = cluster.map_shared_rank(part, lane);
            nb = rp[0]; mb = rp[1]; Mb = rp[2];
        }
        const float n = warp_sum(nb);
        const float mu = warp_sum(nb * mb) / n;
        const float d = mb - mu;
        const float M2 = warp_sum(Mb + nb * d * d);
        if (lane == 0) {
            sm[0] = mu; sm[1] = 1.0f / sqrtf(M2 / n + GN_EPS);
            if (chunk == 0) { stats[(b * GN_G + g) * 2] = sm[0]; stats[(b * GN_G + g) * 2 + 1] = sm[1]; }
        }
    }
    cluster.barrier_arrive();                                // remote reads of `part` are done; waited for before exit
    __syncthreads();
    const float mean = sm[0], rstd = sm[1];
    const float4 sc = make_float4(rstd * ga.x, rstd * ga.y, rstd * ga.z, rstd * ga.w);
#pragma unroll
    for (int i = 0; i < GN_V; ++i) {
        if (ok[i]) {
            float4 o;
            o.x = (v[i].x - mean) * sc.x + be.x; o.y = (v[i].y - mean) * sc.y + be.y;
            o.z = (v[i].z - mean) * sc.z + be.z; o.w = (v[i].w - mean) * sc.w + be.w;
            if (res != nullptr) { o.x += rr[i].x; o.y += rr[i].y; o.z += rr[i].z; o.w += rr[i].w; }
            if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
            *reinterpret_cast<float4*>(out + e0 + i * estep) = o;
        }
    }
    cluster.barrier_wait();
}

int gn_fwd_fused(const float* y, const float* gamma, const float* beta, const float* res, float* out, float* stats, float* partial,
                 int B, int HW, int C, int relu, cudaStream_t st) {
    (void)partial;
    GnPlan pl;
    if (!gn_plan(HW, C, &pl)) return DBOA_ERR_SHAPE;
    return launch_ex(gn_fwd_fused_kernel, dim3(pl.chunks, GN_G, B), dim3(GN_NT), 0, st, dim3(pl.chunks, 1, 1), true, y, gamma, beta, res, out,
                     stats, HW, C, pl.rows, pl.lg, relu);
}

// backward: grid (chunks, 4, B), cluster (chunks, 1, 1)
//   dz = dout * (mask_src > 0), x^ = (y - mean) rstd, q = dz gamma
//   dy = rstd (q - mean_grp(q) - x^ mean_grp(q x^));  dgamma += sum dz x^;  dbeta += sum dz
__global__ void __launch_bounds__(GN_NT, 1) gn_bwd_fused_kernel(const float* __restrict__ dout, const float* __restrict__ mask_src,
                                                             const float* __restrict__ y, const float* __restrict__ stats,
                                                             const float* __restrict__ gamma, float* __restrict__ dy,
                                                             float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                             float* __restrict__ rows_g, float* __restrict__ rows_b, unsigned* pcounters,
                                                             int HW, int C, int R, int lg, int defer) {
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ float red1[64];
    __shared__ float part[2];
    __shared__ float sm[2];
    __shared__ int s_last;
    __shared__ __align__(16) float4 wred[2][32][32];         // [dgamma|dbeta][warp][lane]: per-warp channel-vector partials
    __shared__ __align__(16) float4 chan[2][128];            // this CTA's per-channel-vector sums (read by the cluster)
    pdl_wait();
    pdl_trigger();
    const int chunk = blockIdx.x, g = blockIdx.y, b = blockIdx.z, chunks = gridDim.x, B = gridDim.z, slot = b * GN_G + g;
    const int cg4 = 1 << lg, cgc = cg4 * 4;
    const int r0 = chunk * R, rows = min(R, HW - r0);
    const int cv = threadIdx.x & (cg4 - 1), rt = threadIdx.x >> lg, rstep = GN_NT >> lg;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const size_t e0 = ((size_t)b * HW + r0 + rt) * C + g * cgc + cv * 4;
    const size_t estep = (size_t)rstep * C;
    const float mean = stats[slot * 2], rstd = stats[slot * 2 + 1];
    const float4 ga = ldg4(gamma + g * cgc + cv * 4);
    float4 d[GN_V], xh[GN_V];
    bool ok[GN_V];
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < GN_V; ++i) {
        ok[i] = rt + i * rstep < rows;
        d[i] = ok[i] ? ldg4(dout + e0 + i * estep) : zero;
        xh[i] = ok[i] ? ldg4(y + e0 + i * estep) : zero;
    }
    if (mask_src != nullptr) {
        float4 m[GN_V];
#pragma unroll
        for (int i = 0; i < GN_V; ++i) m[i] = ok[i] ? ldg4(mask_src + e0 + i * estep) : zero;
#pragma unroll
        for (int i = 0; i < GN_V; ++i) {
            d[i].x = m[i].x > 0.f ? d[i].x : 0.f; d[i].y = m[i].y > 0.f ? d[i].y : 0.f;
            d[i].z = m[i].z > 0.f ? d[i].z : 0.f; d[i].w = m[i].w > 0.f ? d[i].w : 0.f;
        }
    }
    float4 dg = zero, db = zero;
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < GN_V; ++i) {                          // rows past the chunk hold d = 0 and contribute nothing
        xh[i] = make_float4((xh[i].x - mean) * rstd, (xh[i].y - mean) * rstd, (xh[i].z - mean) * rstd, (xh[i].w - mean) * rstd);
        const float4 q = make_float4(d[i].x * ga.x, d[i].y * ga.y, d[i].z * ga.z, d[i].w * ga.w);
        dg.x += d[i].x * xh[i].x; dg.y += d[i].y * xh[i].y; dg.z += d[i].z * xh[i].z; dg.w += d[i].w * xh[i].w;
        db.x += d[i].x; db.y += d[i].y; db.z += d[i].z; db.w += d[i].w;
        s1 += (q.x + q.y) + (q.z + q.w);
        s2 += (q.x * xh[i].x + q.y * xh[i].y) + (q.z * xh[i].z + q.w * xh[i].w);
    }
    // per-channel-vector partials: lanes of a warp that share cv (cg4 < 32) combine by shuffles, then one slot per (warp, lane)
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        if (o >= cg4) {
            dg.x += __shfl_xor_sync(0xffffffffu, dg.x, o); dg.y += __shfl_xor_sync(0xffffffffu, dg.y, o);
            dg.z += __shfl_xor_sync(0xffffffffu, dg.z, o); dg.w += __shfl_xor_sync(0xffffffffu, dg.w, o);
            db.x += __shfl_xor_sync(0xffffffffu, db.x, o); db.y += __shfl_xor_sync(0xffffffffu, db.y, o);
            db.z += __shfl_xor_sync(0xffffffffu, db.z, o); db.w += __shfl_xor_sync(0xffffffffu, db.w, o);
        }
    }
    wred[0][wid][lane] = dg; wred[1][wid][lane] = db;
    const float2 ss = block_sum2(s1, s2, red1);              // contains the __syncthreads that publishes wred
    if (threadIdx.x == 0) { part[0] = ss.x; part[1] = ss.y; }
    if (threadIdx.x < 2 * cg4) {                             // channel vector t: sum over the warps that carry it
        const int which = threadIdx.x >= cg4, t = threadIdx.x - which * cg4;
        const int wl = t & 31, wstep = cg4 > 32 ? cg4 >> 5 : 1, w0 = t >> 5;
        float4 a = zero;
        for (int w = w0; w < 32; w += wstep) {
            const float4 p = wred[which][w][wl];
            a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w;
        }
        chan[which][t] = a;
    }
    cluster.sync();
    if (threadIdx.x < 32) {
        float a = 0.f, c = 0.f;
        if (lane < chunks) {
            const float* rp = cluster.map_shared_rank(part, lane);
            a = rp[0]; c = rp[1];
        }
        a = warp_sum(a); c = warp_sum(c);
        if (lane == 0) { sm[0] = a; sm[1] = c; }
    }
    __syncthreads();
    const float invN = 1.0f / ((float)HW * (float)cgc);
    const float m1 = sm[0] * invN, m2 = sm[1] * invN;
#pragma unroll
    for (int i = 0; i < GN_V; ++i) {
        if (ok[i]) {
            float4 o;
            o.x = rstd * (d[i].x * ga.x - m1 - xh[i].x * m2); o.y = rstd * (d[i].y * ga.y - m1 - xh[i].y * m2);
            o.z = rstd * (d[i].z * ga.z - m1 - xh[i].z * m2); o.w = rstd * (d[i].w * ga.w - m1 - xh[i].w * m2);
            *reinterpret_cast<float4*>(dy + e0 + i * estep) = o;
        }
    }
    // affine-parameter gradients: CTA `chunk` owns the channel vectors t = chunk, chunk + chunks, ... and sums them over
    // the cluster in chunk order through distributed shared memory
    {
        const int which = threadIdx.x >> 7, k = threadIdx.x & 127;           // threads 0..255: [dgamma | dbeta] x 128 slots
        const int t = chunk + k * chunks;
        if (threadIdx.x < 256 && t < cg4) {
            float4 a = zero;
            for (int c = 0; c < chunks; ++c) {
                const float4 p = reinterpret_cast<const float4*>(cluster.map_shared_rank(&chan[0][0], c))[which * 128 + t];
                a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w;
            }
            float* dst = (B == 1 ? (which ? dbeta : dgamma) : (which ? rows_b : rows_g) + (size_t)b * C) + g * cgc + t * 4;
            if (B == 1) {
                float4 cur = *reinterpret_cast<float4*>(dst);
                cur.x += a.x; cur.y += a.y; cur.z += a.z; cur.w += a.w;
                *reinterpret_cast<float4*>(dst) = cur;
            } else {
                *reinterpret_cast<float4*>(dst) = a;
            }
        }
    }
    cluster.barrier_arrive();
    if (B > 1 && !defer) {                                   // last CTA of group g (over samples and chunks) adds the rows in order
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned tk = atomicAdd(&pcounters[g], 1u);
            s_last = (tk == (unsigned)(B * chunks) - 1);
            if (s_last) pcounters[g] = 0;
        }
        __syncthreads();
        if (s_last) {
            __threadfence();
            for (int c = threadIdx.x; c < cgc; c += GN_NT) {
                float a = 0.f, bsum = 0.f;
                for (int r = 0; r < B; ++r) { a += __ldcg(rows_g + (size_t)r * C + g * cgc + c); bsum += __ldcg(rows_b + (size_t)r * C + g * cgc + c); }
                dgamma[g * cgc + c] += a; dbeta[g * cgc + c] += bsum;
            }
        }
    }
    cluster.barrier_wait();
}

int gn_bwd_fused(const float* dout, const float* mask_src, const float* y, const float* stats, const float* gamma, float* dy,
                 float* dgamma, float* dbeta, float* partial, int B, int HW, int C, cudaStream_t st, int defer) {
    GnPlan pl;
    if (!gn_plan(HW, C, &pl) || (C / 16) > 128) return DBOA_ERR_SHAPE;
    unsigned* cnt = sync_words();
    if (!cnt) return DBOA_ERR_CUDA;
    return launch_ex(gn_bwd_fused_kernel, dim3(pl.chunks, GN_G, B), dim3(GN_NT), 0, st, dim3(pl.chunks, 1, 1), true, dout, mask_src, y, stats,
                     gamma, dy, dgamma, dbeta, partial, partial + (size_t)B * C, cnt, HW, C, pl.rows, pl.lg, defer);
}

// Deferred affine-parameter gradients of a whole network (B > 1): every GroupNorm backward left its per-sample rows
// [B][C] (dgamma) | [B][C] (dbeta) at rows + 2 * B * item.cum_channels; ONE launch adds them to the gradient arena in sample
// order.  This keeps the per-layer kernels free of the fence + ticket + last-CTA pass that B > 1 otherwise needs.
__global__ void __launch_bounds__(256) gn_param_finish_kernel(const GnFinishItem* __restrict__ items, const float* __restrict__ rows,
                                                              float* __restrict__ G, int B) {
    pdl_wait();
    pdl_trigger();
    const GnFinishItem it = items[blockIdx.x];
    const float* rg = rows + 2 * (size_t)B * it.cum_channels;
    const float* rb = rg + (size_t)B * it.C;
    for (int c = threadIdx.x; c < it.C; c += 256) {
        float a = 0.f, bsum = 0.f;
        for (int r = 0; r < B; ++r) { a += rg[(size_t)r * it.C + c]; bsum += rb[(size_t)r * it.C + c]; }
        G[it.g_off + c] += a; G[it.b_off + c] += bsum;
    }
}

int gn_param_finish(const GnFinishItem* items_dev, int n_items, const float* rows, float* G, int B, cudaStream_t st) {
    return launch_ex(gn_param_finish_kernel, dim3(n_items), dim3(256), 0, st, dim3(1, 1, 1), true, items_dev, rows, G, B);
}

}  // namespace dboa
