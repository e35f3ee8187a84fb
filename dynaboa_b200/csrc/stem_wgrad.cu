// Weight gradient of the 7x7 / stride-2 stem convolution (3 -> 64 channels, 224^2 -> 112^2): reference model/hmr.py:96 `conv1`
// under loss.backward() (dynaboa_benchmark.py:150).
//
// It is the LAST kernel of every backward (its dy exists only after the whole data-gradient chain), so its duration is on the
// critical path of the frame.  As an implicit GEMM it is M = 64 output channels, N = 147 (tap, ci), K = 12544 B pixels: the
// generic CUDA-core kernel has 3 tiles and a 16-CTA cluster split -- 48 CTAs of 49 serial iterations, 81 us at batch 1.  Here
// one CTA owns whole output rows: the 112 x 64 dy row and the 7 zero-padded input rows it touches are staged in shared memory
// once, thread (co, q) keeps 19 of the 147 accumulators of its output channel in registers (operand reads are warp-wide
// broadcasts), and the per-CTA partials [64][147] go to a workspace that a second small launch adds into the gradient arena in
// a fixed order (deterministic).  112 CTAs at batch 1.
#include <stdint.h>

#include "common.cuh"
#include "kernels.h"

namespace dboa {
namespace stem {

constexpr int CO = 64, KK = 147, HO = 112, HI = 224, ROWF = (HI + 6) * 3;      // 690 floats per zero-padded input row
constexpr int NT = 512, JPT = 19;                                               // 8 thread groups x 19 accumulators (the last one 14)
constexpr int SMEM_FLOATS = HO * CO + 7 * ROWF;                                 // 7168 + 4830 (>= 64 * 147 for the transpose)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
template <int IMM>
__device__ __forceinline__ float lds_imm(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(a), "n"(IMM));
    return v;
}

__global__ void __launch_bounds__(NT) stem_wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ part,
                                                        int B, int rows_per_cta) {
    extern __shared__ __align__(16) float sm[];
    float* dys = sm;                        // [112][64]
    float* xs = sm + HO * CO;               // [7][ROWF]: xs[r][(wi + 3) * 3 + ci], rows hi = 2 ho - 3 + r
    const int tid = threadIdx.x, co = tid & 63, q = tid >> 6;
    const int j0 = q * JPT, nj = min(JPT, KK - j0);
    uint32_t addr[JPT];                     // shared address of x for (tap, ci) = j0 + jj at output column 0
    const uint32_t xs32 = smem_u32(xs), dys32 = smem_u32(dys) + (uint32_t)co * 4u;
#pragma unroll
    for (int jj = 0; jj < JPT; ++jj) {
        const int j = min(j0 + jj, KK - 1), r = j / 21;
        addr[jj] = xs32 + (uint32_t)(r * ROWF + (j - r * 21)) * 4u;
    }
    float acc[JPT];
#pragma unroll
    for (int jj = 0; jj < JPT; ++jj) acc[jj] = 0.f;
    pdl_wait();
    pdl_trigger();
    const int total_rows = B * HO;
    const int row_begin = blockIdx.x * rows_per_cta, row_end = min(total_rows, row_begin + rows_per_cta);
    for (int row = row_begin; row < row_end; ++row) {
        const int b = row / HO, ho = row - b * HO;
        __syncthreads();
        const float4* src = reinterpret_cast<const float4*>(dy + ((size_t)b * HO + ho) * HO * CO);
        for (int i = tid; i < HO * CO / 4; i += NT) reinterpret_cast<float4*>(dys)[i] = __ldcg(src + i);
        for (int i = tid; i < 7 * ROWF; i += NT) {
            const int r = i / ROWF, c = i - r * ROWF, hi = 2 * ho - 3 + r, w3 = c - 9;
            float v = 0.f;
            if ((unsigned)hi < (unsigned)HI && (unsigned)w3 < (unsigned)(HI * 3)) v = __ldg(x + ((size_t)b * HI + hi) * (HI * 3) + w3);
            xs[i] = v;
        }
        __syncthreads();
#pragma unroll 1
        for (int wo = 0; wo < HO; wo += 4) {                 // 4 output columns per trip: x addresses advance by 6 floats each
            float d[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) d[u] = lds_imm<0>(dys32 + (uint32_t)((wo + u) * CO) * 4u);
            const uint32_t step = (uint32_t)wo * 24u;
#pragma unroll
            for (int jj = 0; jj < JPT; ++jj) {
                const uint32_t a = addr[jj] + step;
                acc[jj] = fmaf(d[0], lds_imm<0>(a), acc[jj]);
                acc[jj] = fmaf(d[1], lds_imm<24>(a), acc[jj]);
                acc[jj] = fmaf(d[2], lds_imm<48>(a), acc[jj]);
                acc[jj] = fmaf(d[3], lds_imm<72>(a), acc[jj]);
            }
        }
    }
    __syncthreads();
    float* outs = sm;                       // [64][147]
#pragma unroll
    for (int jj = 0; jj < JPT; ++jj)
        if (jj < nj) outs[co * KK + j0 + jj] = acc[jj];
    __syncthreads();
    float* dst = part + (size_t)blockIdx.x * (CO * KK);
    for (int i = tid; i < CO * KK; i += NT) dst[i] = outs[i];
}

__global__ void __launch_bounds__(256) stem_wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, int nparts, int kpitch) {
    pdl_wait();
    pdl_trigger();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= CO * KK) return;
    float s0 = 0.f, s1 = 0.f;
    int c = 0;
    for (; c + 1 < nparts; c += 2) { s0 += __ldcg(part + (size_t)c * (CO * KK) + i); s1 += __ldcg(part + (size_t)(c + 1) * (CO * KK) + i); }
    if (c < nparts) s0 += __ldcg(part + (size_t)c * (CO * KK) + i);
    const int co = i / KK, j = i - co * KK;
    dw[(size_t)co * kpitch + j] += s0 + s1;
}

}  // namespace stem

bool stem_wgrad_ok(const ConvDims& d) {
    return d.Cin == 3 && d.Cout == stem::CO && d.kh == 7 && d.kw == 7 && d.stride == 2 && d.pad == 3 && d.Hi == stem::HI && d.Wi == stem::HI &&
           d.Ho == stem::HO && d.Wo == stem::HO && d.Kpitch >= stem::KK;
}

int stem_wgrad(const float* dy, const float* x, float* dw, const ConvDims& d, float* ws, size_t ws_floats, cudaStream_t st) {
    if (!stem_wgrad_ok(d)) return DBOA_ERR_UNSUPPORTED;
    const int rows = d.B * stem::HO;
    const int max_parts = (int)std::min<size_t>(2 * num_sms(), ws_floats / (stem::CO * stem::KK));
    if (ws == nullptr || max_parts < 1) return DBOA_ERR_UNSUPPORTED;
    const int rows_per = ceil_div(rows, max_parts), nparts = ceil_div(rows, rows_per);
    DBOA_TRY(launch_ex(stem::stem_wgrad_kernel, dim3(nparts), dim3(stem::NT), (size_t)stem::SMEM_FLOATS * sizeof(float), st, dim3(1, 1, 1), true,
                       dy, x, ws, d.B, rows_per));
    return launch_ex(stem::stem_wgrad_reduce_kernel, dim3(ceil_div(stem::CO * stem::KK, 256)), dim3(256), 0, st, dim3(1, 1, 1), true,
                     (const float*)ws, dw, nparts, d.Kpitch);
}

}  // namespace dboa
