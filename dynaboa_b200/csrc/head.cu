// Iterative regressor head: small-batch linear layers (weight-streaming GEMV class) forward,
// data gradient and weight gradient, plus the 6D -> rotation-matrix map.
//
// Replaces the cuBLAS calls behind reference model/hmr.py:158-172 (fc1/fc2/decpose/decshape/deccam,
// 3 iterations) and utils/geometry.py:47-61 (rot6d_to_rotmat) -- SURVEY.md §2.1 K4/K5.
#include "common.cuh"
#include "kernels.h"
#include "rotmath.cuh"

namespace dboa {

// ---------------------------------------------------------------------------------------------
// forward: FOUR warps per output neuron (each a quarter of K, all its loads in flight at once), two neurons per
// CTA, up to 8 batch rows per pass.  At batch 1-3 this is a weight-streaming GEMV whose time is the number of
// dependent load round trips per warp, not bytes: one warp per neuron walked K in 17 serial steps.
// ---------------------------------------------------------------------------------------------
template <int BT>
__global__ void __launch_bounds__(256) linear_fwd_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ W, int ldw,
                                                         const float* __restrict__ bias, const float* __restrict__ addend, int ld_add,
                                                         const float* __restrict__ mask, float* __restrict__ pre,
                                                         float* __restrict__ post, int ld_out, float* __restrict__ post2, int ld_out2,
                                                         int b0, int nb, int N, int K, int bper, long long wstride,
                                                         unsigned long long active) {
    __shared__ float sred[8][BT];
    if (!((active >> blockIdx.y) & 1ULL)) return;           // grouped: an idle group's rows are not computed
    pdl_wait();
    pdl_trigger();
    b0 += blockIdx.y * bper;                                // grouped: rows of group blockIdx.y, its own weights
    W += blockIdx.y * wstride;
    if (bias) bias += blockIdx.y * wstride;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, part = warp & 3;
    const int n = blockIdx.x * 2 + (warp >> 2);
    float acc[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[b] = 0.f;
    if (n < N) {
        const float* wr = W + (size_t)n * ldw;
        const bool vec = ((ldw & 3) == 0) && ((ldx & 3) == 0);
        int kdone = 0;
        if (vec) {
            const int K4 = K >> 2, per = (K4 + 3) >> 2;
            const int kbeg = part * per, kend = min(K4, kbeg + per);
            for (int base = kbeg; base < kend; base += 160) {          // 5 float4 per lane and pass, issued together
                float4 wv[5];
#pragma unroll
                for (int i = 0; i < 5; ++i) {
                    const int k4 = base + lane + 32 * i;
                    wv[i] = k4 < kend ? ldg4(wr + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int b = 0; b < BT; ++b)
                    if (b < nb) {
                        float4 xv[5];
#pragma unroll
                        for (int i = 0; i < 5; ++i) {
                            const int k4 = base + lane + 32 * i;
                            xv[i] = k4 < kend ? ldg4(x + (size_t)(b0 + b) * ldx + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                        }
#pragma unroll
                        for (int i = 0; i < 5; ++i)
                            acc[b] += (wv[i].x * xv[i].x + wv[i].y * xv[i].y) + (wv[i].z * xv[i].z + wv[i].w * xv[i].w);
                    }
            }
            kdone = K4 * 4;
        }
        // scalar remainder (K % 4, or everything when the pitches are not 16-byte multiples): split over the four warps too
        for (int k = kdone + part * 32 + lane; k < K; k += 128) {
            const float wv = __ldg(wr + k);
#pragma unroll
            for (int b = 0; b < BT; ++b)
                if (b < nb) acc[b] += wv * __ldg(x + (size_t)(b0 + b) * ldx + k);
        }
    }
#pragma unroll
    for (int b = 0; b < BT; ++b) {
        acc[b] = warp_sum(acc[b]);
        if (lane == 0) sred[warp][b] = acc[b];
    }
    __syncthreads();
    if (n < N && part == 0 && lane < nb) {                 // lane b finishes batch row b: the four K-quarters in fixed order
        const int b = lane, bb = b0 + b;
        float y = ((sred[warp][b] + sred[warp + 1][b]) + (sred[warp + 2][b] + sred[warp + 3][b])) + (bias ? bias[n] : 0.f);
        if (addend) y += addend[(size_t)bb * ld_add + n];
        if (pre) pre[(size_t)bb * ld_out + n] = y;
        const float m = mask ? mask[(size_t)bb * N + n] : 1.0f;
        const float o = y * m;
        if (post) post[(size_t)bb * ld_out + n] = o;
        if (post2) post2[(size_t)bb * ld_out2 + n] = o;
    }
}

int linear_fwd(const float* x, int ldx, const float* W, int ldw, const float* bias, const float* addend, int ld_add, const float* mask,
               float* pre, float* post, int ld_out, float* post2, int ld_out2, int B, int N, int K, cudaStream_t st, int groups,
               long long wstride, unsigned long long active) {
    if (groups < 1 || B % groups != 0) return DBOA_ERR_SHAPE;
    const int bper = B / groups;
    for (int b0 = 0; b0 < bper; b0 += 8) {
        int nb = bper - b0 < 8 ? bper - b0 : 8;
        DBOA_TRY(launch_ex(linear_fwd_kernel<8>, dim3(ceil_div(N, 2), groups), dim3(256), 0, st, dim3(1, 1, 1), true, x, ldx, W, ldw, bias, addend, ld_add, mask, pre, post, ld_out, post2, ld_out2, b0, nb, N, K, bper, wstride, active));
    }
    return DBOA_OK;
}

// ---------------------------------------------------------------------------------------------
// data gradient: dx[b][k] = sum_n dy[b][n] W[n][k]; grid (ceil(K/256), nsplit), fixed-order reduce
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) linear_dgrad_kernel(const float* __restrict__ dy, int ldy, const float* __restrict__ W, int ldw,
                                                           float* __restrict__ part, int b0, int nb, int B, int N, int K, int nlen,
                                                           int bper, long long wstride, unsigned long long active) {
    if (!((active >> blockIdx.z) & 1ULL)) return;           // grouped: an idle group's partial rows are not computed
    pdl_wait();
    pdl_trigger();
    b0 += blockIdx.z * bper;                                // grouped: rows of group blockIdx.z, its own weights
    W += blockIdx.z * wstride;
    __shared__ float sdy[8][128];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int nbeg = blockIdx.y * nlen, nend = min(nbeg + nlen, N);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int n0 = nbeg; n0 < nend; n0 += 128) {
        const int cnt = min(128, nend - n0);
        __syncthreads();
        for (int i = threadIdx.x; i < 8 * 128; i += 256) {
            int b = i >> 7, j = i & 127;
            sdy[b][j] = (b < nb && j < cnt) ? dy[(size_t)(b0 + b) * ldy + n0 + j] : 0.f;
        }
        __syncthreads();
        if (k < K) {
#pragma unroll 8
            for (int j = 0; j < cnt; ++j) {
                float wv = __ldg(W + (size_t)(n0 + j) * ldw + k);
#pragma unroll
                for (int b = 0; b < 8; ++b) acc[b] = fmaf(sdy[b][j], wv, acc[b]);
            }
        }
    }
    if (k < K)
        for (int b = 0; b < nb; ++b) part[((size_t)blockIdx.y * B + b0 + b) * K + k] = acc[b];
}

__global__ void linear_dgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dx, int ldx, int B, int K, int nsplit) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * K) return;
    int b = i / K, k = i - b * K;
    float s = 0.f;
#pragma unroll 8
    for (int z = 0; z < nsplit; ++z) s += part[((size_t)z * B + b) * K + k];
    dx[(size_t)b * ldx + k] = s;
}

int linear_dgrad(const float* dy, int ldy, const float* W, int ldw, float* dx, int ldx, int B, int N, int K, float* ws, size_t ws_floats,
                 cudaStream_t st, int groups, long long wstride, unsigned long long active) {
    if (groups < 1 || B % groups != 0) return DBOA_ERR_SHAPE;
    const int bper = B / groups;
    // 32 rows of W per CTA: at batch 1-3 the kernel is a chain of dependent weight loads, so many short CTAs beat few long ones
    int nsplit = ceil_div(N, 32);
    while (nsplit > 1 && (size_t)nsplit * B * K > ws_floats) nsplit = (nsplit + 1) >> 1;
    if ((size_t)nsplit * B * K > ws_floats) return DBOA_ERR_ARG;
    int nlen = ceil_div(N, nsplit);
    nlen = (nlen + 31) / 32 * 32;
    nsplit = ceil_div(N, nlen);
    for (int b0 = 0; b0 < bper; b0 += 8) {
        int nb = bper - b0 < 8 ? bper - b0 : 8;
        dim3 grid(ceil_div(K, 256), nsplit, groups);
        DBOA_TRY(launch_ex(linear_dgrad_kernel, dim3(grid), dim3(256), 0, st, dim3(1, 1, 1), true, dy, ldy, W, ldw, ws, b0, nb, B, N, K, nlen,
                           bper, wstride, active));
    }
    return launch_ex(linear_dgrad_reduce_kernel, dim3(ceil_div(B * K, 256)), dim3(256), 0, st, dim3(1, 1, 1), true, ws, dx, ldx, B, K, nsplit);
}

// ---------------------------------------------------------------------------------------------
// weight gradient: dW[n][k] += sum_r dy[r][n] x[r][k]; db[n] += sum_r dy[r][n]; R <= 32 rows
// ---------------------------------------------------------------------------------------------
// Grouped (gridDim.z groups): group g reduces its R rows r -> slab r / bper, row g * bper + r % bper of the slab (bstride rows
// apart), in order, into its own dW / db.  One group (GROUPED = false): the rows in memory order.
template <bool GROUPED>
__global__ void __launch_bounds__(256) linear_wgrad_kernel(const float* __restrict__ dy, int ldy, const float* __restrict__ x, int ldx,
                                                           float* __restrict__ dW, int ldw, float* __restrict__ db, int R, int N, int K,
                                                           int bper, int bstride, long long wstride,
                                                           unsigned long long active) {
    const int g = blockIdx.z;
    if (GROUPED && !((active >> g) & 1ULL)) return;         // nothing is added to an idle group's gradient
    pdl_wait();
    pdl_trigger();
    __shared__ float sdy[64];
    const int n = blockIdx.y;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (GROUPED) {
        dW += g * wstride;
        if (db != nullptr) db += g * wstride;
    }
    auto row = [&](int r) {
        if (!GROUPED) return (size_t)r;
        const int slab = r / bper;
        return (size_t)slab * bstride + g * bper + (r - slab * bper);
    };
    float acc = 0.f, bacc = 0.f;
    for (int r0 = 0; r0 < R; r0 += 64) {
        const int cnt = min(64, R - r0);
        __syncthreads();
        if (threadIdx.x < cnt) sdy[threadIdx.x] = dy[row(r0 + threadIdx.x) * ldy + n];
        __syncthreads();
        for (int r = 0; r < cnt; ++r) {
            if (k < K) acc = fmaf(sdy[r], __ldg(x + row(r0 + r) * ldx + k), acc);
            bacc += sdy[r];
        }
    }
    if (k < K) dW[(size_t)n * ldw + k] += acc;
    if (db != nullptr && blockIdx.x == 0 && threadIdx.x == 0) db[n] += bacc;
}

int linear_wgrad(const float* dy, int ldy, const float* x, int ldx, float* dW, int ldw, float* db, int R, int N, int K, cudaStream_t st,
                 int groups, int B, long long wstride, unsigned long long active) {
    int bper = R, bstride = R, rows = R;
    if (groups != 1) {
        if (groups < 1 || B < 1 || B % groups != 0 || R % B != 0) return DBOA_ERR_SHAPE;
        bper = B / groups; bstride = B; rows = R / groups;
    }
    dim3 grid(ceil_div(K, 256), N, groups);
    return launch_ex(groups > 1 ? linear_wgrad_kernel<true> : linear_wgrad_kernel<false>, dim3(grid), dim3(256), 0, st, dim3(1, 1, 1), true,
                     dy, ldy, x, ldx, dW, ldw, db, rows, N, K, bper, bstride, wstride, active);
}

// ---------------------------------------------------------------------------------------------
__global__ void rot6d_fwd_kernel(const float* __restrict__ x, float* __restrict__ R, int n) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float xi[6], Ri[9];
    for (int k = 0; k < 6; ++k) xi[k] = x[(size_t)i * 6 + k];
    rot6d_fwd(xi, Ri);
    for (int k = 0; k < 9; ++k) R[(size_t)i * 9 + k] = Ri[k];
}
__global__ void rot6d_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dR, float* __restrict__ dx, int n) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float xi[6], gi[9], di[6];
    for (int k = 0; k < 6; ++k) xi[k] = x[(size_t)i * 6 + k];
    for (int k = 0; k < 9; ++k) gi[k] = dR[(size_t)i * 9 + k];
    rot6d_bwd(xi, gi, di);
    for (int k = 0; k < 6; ++k) dx[(size_t)i * 6 + k] = di[k];
}
int rot6d_fwd_launch(const float* pose6d, float* rotmat, int n, cudaStream_t st) {
    return launch_ex(rot6d_fwd_kernel, dim3(ceil_div(n, 128)), dim3(128), 0, st, dim3(1, 1, 1), true, pose6d, rotmat, n);
}
int rot6d_bwd_launch(const float* pose6d, const float* drot, float* dpose, int n, cudaStream_t st) {
    return launch_ex(rot6d_bwd_kernel, dim3(ceil_div(n, 128)), dim3(128), 0, st, dim3(1, 1, 1), true, pose6d, drot, dpose, n);
}

__global__ void ew_mul_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o, size_t n) {
    pdl_wait();
    pdl_trigger();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) o[i] = a[i] * b[i];
}
int ew_mul(const float* a, const float* b, float* out, size_t n, cudaStream_t st) {
    return launch_ex(ew_mul_kernel, dim3(ceil_div(n, 256)), dim3(256), 0, st, dim3(1, 1, 1), true, a, b, out, n);
}
// dst[b][j] = a[b][j] + b[b][j] for j < n
__global__ void ew_add_rows_kernel(float* dst, int ld_dst, const float* a, int lda, const float* b, int ldb, int B, int n) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * n) return;
    int r = i / n, j = i - r * n;
    dst[(size_t)r * ld_dst + j] = a[(size_t)r * lda + j] + b[(size_t)r * ldb + j];
}
int ew_add_rows(float* dst, int ld_dst, const float* a, int lda, const float* b, int ldb, int B, int n, cudaStream_t st) {
    return launch_ex(ew_add_rows_kernel, dim3(ceil_div(B * n, 256)), dim3(256), 0, st, dim3(1, 1, 1), true, dst, ld_dst, a, lda, b, ldb, B, n);
}

}  // namespace dboa
