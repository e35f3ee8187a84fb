// ReLU masks, max / average pooling and the NCHW -> NHWC input transpose on NHWC fp32 activations.
//
// Replaces the ATen kernels behind reference model/hmr.py:36/57-58 (ReLU backward), :75 (MaxPool2d(3,2,1)),
// :80 (AvgPool2d(7)) -- SURVEY.md section 2.1 K3.  GroupNorm lives in groupnorm.cu.
#include "common.cuh"
#include "kernels.h"

namespace dboa {
// ---------------------------------------------------------------------------------------------
__global__ void relu_mask_kernel(const float* __restrict__ dout, const float* __restrict__ mask_src, float* __restrict__ dz, size_t n4) {
    pdl_wait();
    pdl_trigger();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 d = ldg4(dout + i * 4), m = ldg4(mask_src + i * 4);
    d.x = m.x > 0.f ? d.x : 0.f; d.y = m.y > 0.f ? d.y : 0.f; d.z = m.z > 0.f ? d.z : 0.f; d.w = m.w > 0.f ? d.w : 0.f;
    *reinterpret_cast<float4*>(dz + i * 4) = d;
}
int relu_mask(const float* dout, const float* mask_src, float* dz, size_t n, cudaStream_t st) {
    return launch_ex(relu_mask_kernel, dim3(ceil_div(n / 4, 256)), dim3(256), 0, st, dim3(1, 1, 1), true, dout, mask_src, dz, n / 4);
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int HW, size_t total) {
    pdl_wait();
    pdl_trigger();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;      // over B*HW pixels
    if (i >= total) return;
    size_t b = i / HW, p = i - b * HW;
    for (int c = 0; c < C; ++c) y[i * C + c] = __ldg(x + (b * C + c) * HW + p);
}
int nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, cudaStream_t st) {
    size_t total = (size_t)B * H * W;
    return launch_ex(nchw_to_nhwc_kernel, dim3(ceil_div(total, 256)), dim3(256), 0, st, dim3(1, 1, 1), false, x, y, C, H * W, total);
}

// MaxPool2d(kernel 3, stride 2, pad 1); first maximum in (row, col) scan order wins, as ATen does.
__global__ void maxpool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned char* __restrict__ idx, int B, int H,
                                   int W, int C) {
    pdl_wait();
    pdl_trigger();
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)B * Ho * Wo * C4;
    if (i >= total) return;
    int cv = (int)(i % C4);
    size_t p = i / C4;
    int wo = (int)(p % Wo); p /= Wo;
    int ho = (int)(p % Ho);
    int b = (int)(p / Ho);
    float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    unsigned char bi[4] = {0, 0, 0, 0};
    for (int r = 0; r < 3; ++r) {
        int hi = ho * 2 - 1 + r;
        if ((unsigned)hi >= (unsigned)H) continue;
        for (int s = 0; s < 3; ++s) {
            int wi = wo * 2 - 1 + s;
            if ((unsigned)wi >= (unsigned)W) continue;
            float4 v = ldg4(x + (((size_t)b * H + hi) * W + wi) * C + cv * 4);
            float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (vv[e] > best[e] || vv[e] != vv[e]) { best[e] = vv[e]; bi[e] = (unsigned char)(r * 3 + s); }
        }
    }
    size_t o = (((size_t)b * Ho + ho) * Wo + wo) * C + cv * 4;
    *reinterpret_cast<float4*>(y + o) = make_float4(best[0], best[1], best[2], best[3]);
    *reinterpret_cast<uchar4*>(idx + o) = make_uchar4(bi[0], bi[1], bi[2], bi[3]);
}
// The kernels take even H and W (output H/2 x W/2, which is MaxPool2d(3, 2, 1)'s (H + 1) / 2 only for even extents) and whole
// float4 channel vectors (C % 4 == 0); any other shape is refused rather than computed with a row, a column or channels missing.
static bool maxpool_shape_ok(int H, int W, int C) { return ((H | W) & 1) == 0 && C % 4 == 0; }

int maxpool3x3s2_fwd(const float* x, float* y, unsigned char* idx, int B, int H, int W, int C, cudaStream_t st) {
    if (!maxpool_shape_ok(H, W, C)) return DBOA_ERR_SHAPE;
    size_t total = (size_t)B * (H / 2) * (W / 2) * (C / 4);
    return launch_ex(maxpool_fwd_kernel, dim3(ceil_div(total, 256)), dim3(256), 0, st, dim3(1, 1, 1), true, x, y, idx, B, H, W, C);
}

__global__ void maxpool_bwd_kernel(const float* __restrict__ dy, const unsigned char* __restrict__ idx, float* __restrict__ dx, int B,
                                   int H, int W, int C) {
    pdl_wait();
    pdl_trigger();
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)B * H * W * C4;
    if (i >= total) return;
    int cv = (int)(i % C4);
    size_t p = i / C4;
    int wi = (int)(p % W); p /= W;
    int hi = (int)(p % H);
    int b = (int)(p / H);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ho = hi / 2; ho <= (hi + 1) / 2; ++ho) {
        if (ho >= Ho) continue;
        int r = hi - (ho * 2 - 1);
        if (r < 0 || r > 2) continue;
        for (int wo = wi / 2; wo <= (wi + 1) / 2; ++wo) {
            if (wo >= Wo) continue;
            int s = wi - (wo * 2 - 1);
            if (s < 0 || s > 2) continue;
            size_t o = (((size_t)b * Ho + ho) * Wo + wo) * C + cv * 4;
            uchar4 k = *reinterpret_cast<const uchar4*>(idx + o);
            float4 g = ldg4(dy + o);
            unsigned char me = (unsigned char)(r * 3 + s);
            if (k.x == me) acc[0] += g.x;
            if (k.y == me) acc[1] += g.y;
            if (k.z == me) acc[2] += g.z;
            if (k.w == me) acc[3] += g.w;
        }
    }
    *reinterpret_cast<float4*>(dx + (((size_t)b * H + hi) * W + wi) * C + cv * 4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
}
int maxpool3x3s2_bwd(const float* dy, const unsigned char* idx, float* dx, int B, int H, int W, int C, cudaStream_t st) {
    if (!maxpool_shape_ok(H, W, C)) return DBOA_ERR_SHAPE;
    size_t total = (size_t)B * H * W * (C / 4);
    return launch_ex(maxpool_bwd_kernel, dim3(ceil_div(total, 256)), dim3(256), 0, st, dim3(1, 1, 1), true, dy, idx, dx, B, H, W, C);
}

__global__ void avgpool_fwd_kernel(const float* __restrict__ x, float* __restrict__ out, int HW, int C, int ld, int ncopy,
                                   size_t copy_stride, int total) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int b = i / C, c = i - b * C;
    float s = 0.f;
    for (int p = 0; p < HW; ++p) s += __ldg(x + ((size_t)b * HW + p) * C + c);
    s = s / (float)HW;
    for (int k = 0; k < ncopy; ++k) out[k * copy_stride + (size_t)b * ld + c] = s;
}
int avgpool_fwd(const float* x, float* out, int B, int HW, int C, int ld, int ncopy, size_t copy_stride, cudaStream_t st) {
    return launch_ex(avgpool_fwd_kernel, dim3(ceil_div(B * C, 256)), dim3(256), 0, st, dim3(1, 1, 1), true, x, out, HW, C, ld, ncopy, copy_stride, B * C);
}

__global__ void avgpool_bwd_kernel(const float* __restrict__ dxf, int ld, float* __restrict__ dx, int HW, int C, size_t total) {
    pdl_wait();
    pdl_trigger();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int c = (int)(i % C);
    size_t b = i / ((size_t)HW * C);
    dx[i] = dxf[b * ld + c] / (float)HW;
}
int avgpool_bwd(const float* dxf, int ld, float* dx, int B, int HW, int C, cudaStream_t st) {
    size_t total = (size_t)B * HW * C;
    return launch_ex(avgpool_bwd_kernel, dim3(ceil_div(total, 256)), dim3(256), 0, st, dim3(1, 1, 1), true, dxf, ld, dx, HW, C, total);
}

}  // namespace dboa
