// Input side of the hot path on the GPU: bounding-box crop (zero fill outside the frame) + anti-aliased bilinear resize to
// 224 x 224 + /255 + per-channel normalisation + HWC -> CHW, and the integer keypoint transform.
//
// Replaces reference utils/dataprocess.py:48-96 (crop with skimage.transform.resize), boa_dataset/pw3d.py:127-136,144-149
// (rgb_processing, Normalize) and :151-163 + utils/dataprocess.py:13-46 (j2d_processing / transform) for the benchmark path
// (rot = 0, no flip).  skimage's resize is linear and separable (Gaussian pre-filter, then order-1 zoom, mirror boundaries),
// so   out = Wy . crop . Wx^T   with banded matrices the host composes once per crop size (dataprocess.py); the two kernels
// below apply them: an HBM-streaming pass over the crop rows, then a 224 x 224 x 3 pass.
#include "common.cuh"
#include "kernels.h"

namespace dboa {

// tmp[yc][xo][c] = sum_j wx[xo][j] * crop(yc, sx[xo] + j, c);  crop(y, x) = img(ul_y + y, ul_x + x) or 0 outside the frame.
// Element i = yc * res + xo of one frame.
template <typename T>
__device__ __forceinline__ void crop_rows_elem(const T* __restrict__ img, int H, int W, int ul_x, int ul_y, const float* __restrict__ wx,
                                               const int* __restrict__ sx, int Tx, int res, int i, float* __restrict__ tmp) {
    const int yc = i / res, xo = i - yc * res, y = ul_y + yc;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    if (y >= 0 && y < H) {
        const int x0 = ul_x + sx[xo];
        const float* w = wx + (size_t)xo * Tx;
        const T* row = img + (size_t)y * W * 3;
        for (int j = 0; j < Tx; ++j) {
            const int x = x0 + j;
            if (x >= 0 && x < W) {
                const float wj = __ldg(w + j);
                a0 = fmaf(wj, (float)row[x * 3 + 0], a0); a1 = fmaf(wj, (float)row[x * 3 + 1], a1); a2 = fmaf(wj, (float)row[x * 3 + 2], a2);
            }
        }
    }
    float* o = tmp + (size_t)i * 3;
    o[0] = a0; o[1] = a1; o[2] = a2;
}
// out[c][yo][xo] = ((sum_i wy[yo][i] * tmp[sy[yo] + i][xo][c]) / 255 - mean[c]) / std[c];  element i = yo * res + xo of one frame
__device__ __forceinline__ void crop_cols_elem(const float* __restrict__ tmp, int Hc, const float* __restrict__ wy, const int* __restrict__ sy,
                                               int Ty, int res, float m0, float m1, float m2, float s0, float s1, float s2, int i,
                                               float* __restrict__ out) {
    const int yo = i / res, xo = i - yo * res;
    const float* w = wy + (size_t)yo * Ty;
    const int y0 = sy[yo];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int k = 0; k < Ty; ++k) {
        const int y = y0 + k;
        if (y >= 0 && y < Hc) {
            const float wk = __ldg(w + k);
            const float* t = tmp + ((size_t)y * res + xo) * 3;
            a0 = fmaf(wk, t[0], a0); a1 = fmaf(wk, t[1], a1); a2 = fmaf(wk, t[2], a2);
        }
    }
    const size_t plane = (size_t)res * res;
    out[i] = __fdiv_rn(__fsub_rn(__fdiv_rn(a0, 255.0f), m0), s0);
    out[plane + i] = __fdiv_rn(__fsub_rn(__fdiv_rn(a1, 255.0f), m1), s1);
    out[2 * plane + i] = __fdiv_rn(__fsub_rn(__fdiv_rn(a2, 255.0f), m2), s2);
}
// utils/dataprocess.py:39-46 applied to kp + 1 (pw3d.py:155): p = t . (x, y, 1) in double, truncation toward zero, + 1, then
// 2 p / res - 1 (double) -> float; the confidence column is copied.  One keypoint: the body of keypoint_transform_kernel and of
// the grouped call.
__device__ __forceinline__ void keypoint_elem(const float* __restrict__ k, double t00, double t02, double t11, double t12, int res,
                                              float* __restrict__ o) {
    const double x = (double)k[0] + 1.0 - 1.0, y = (double)k[1] + 1.0 - 1.0;
    const double px = (double)((int)(t00 * x + t02) + 1), py = (double)((int)(t11 * y + t12) + 1);
    o[0] = (float)(2.0 * px / res - 1.0);
    o[1] = (float)(2.0 * py / res - 1.0);
    o[2] = k[2];
}
__global__ void keypoint_transform_kernel(const float* __restrict__ kp, int n, double t00, double t02, double t11, double t12, int res,
                                          float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keypoint_elem(kp + i * 3, t00, t02, t11, t12, res, out + i * 3);
}
int keypoint_transform(const float* kp, int n, double t00, double t02, double t11, double t12, int res, float* out, cudaStream_t st) {
    if (n < 1) return DBOA_OK;
    keypoint_transform_kernel<<<ceil_div(n, 128), 128, 0, st>>>(kp, n, t00, t02, t11, t12, res, out);
    return check_launch();
}

// ---- grouped input side: the frames of several streams in one launch per pass.  The descriptors of the active videos travel
// compacted in the kernel parameter (__grid_constant__: read in place from parameter space, no host-to-device copy); entry k
// describes video video[k].  Per element the arithmetic is crop_rows_elem / crop_cols_elem / keypoint_elem, so each active
// row is bit-identical to the one-frame call (for the crop, this call with a single entry).
struct CropGroups {
    dboa_crop_desc f[64];
    long long tmp_off[64];        // float offset of entry k's rows in tmp
    int first_block[65];          // rows pass: blocks [first_block[k], first_block[k + 1]) belong to entry k
    unsigned char video[64];
    int n, res;
    float mean[3], stdv[3];
};

// one row of blocks per entry, back to back: entry k's blocks see exactly the indices of a grid of its own
__global__ void __launch_bounds__(256) crop_groups_rows_kernel(const __grid_constant__ CropGroups a, float* __restrict__ tmp) {
    int lo = 0, hi = a.n - 1;                                         // last entry whose first block is <= blockIdx.x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.first_block[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const dboa_crop_desc& f = a.f[lo];
    const int i = ((int)blockIdx.x - a.first_block[lo]) * blockDim.x + threadIdx.x;
    if (i >= f.Hc * a.res) return;
    float* t = tmp + a.tmp_off[lo];
    if (f.is_u8)
        crop_rows_elem(static_cast<const unsigned char*>(f.img), f.H, f.W, f.ul_x, f.ul_y, f.wx, f.sx, f.Tx, a.res, i, t);
    else
        crop_rows_elem(static_cast<const float*>(f.img), f.H, f.W, f.ul_x, f.ul_y, f.wx, f.sx, f.Tx, a.res, i, t);
}
// grid row k: entry k's res * res outputs into its video's row of out
__global__ void __launch_bounds__(256) crop_groups_cols_kernel(const __grid_constant__ CropGroups a, const float* __restrict__ tmp,
                                                               float* __restrict__ out) {
    const int k = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.res * a.res) return;
    const dboa_crop_desc& f = a.f[k];
    crop_cols_elem(tmp + a.tmp_off[k], f.Hc, f.wy, f.sy, f.Ty, a.res, a.mean[0], a.mean[1], a.mean[2], a.stdv[0], a.stdv[1], a.stdv[2], i,
                   out + (size_t)a.video[k] * 3 * a.res * a.res);
}

// bit g of `active` set and g < groups; a nonzero mask
static bool mask_ok(int groups, unsigned long long active) { return active != 0 && (groups >= 64 || (active >> groups) == 0); }

int crop_resize_normalize_groups(const dboa_crop_desc* frames, int groups, unsigned long long active, int res, const float mean[3],
                                 const float stdv[3], float* tmp, long long tmp_floats, float* out, cudaStream_t st) {
    if (groups < 1 || groups > 64 || res < 1) return DBOA_ERR_SHAPE;
    if (!mask_ok(groups, active)) return DBOA_ERR_ARG;
    CropGroups a;
    a.n = 0; a.res = res;
    long long need = 0, blocks = 0;
    for (int g = 0; g < groups; ++g) {
        if (!((active >> g) & 1ULL)) continue;
        const dboa_crop_desc& f = frames[g];
        if (!f.img || !f.wx || !f.sx || !f.wy || !f.sy) return DBOA_ERR_ARG;
        if (f.H < 1 || f.W < 1 || f.Hc < 1 || f.Tx < 1 || f.Ty < 1) return DBOA_ERR_SHAPE;
        const int k = a.n++;
        a.f[k] = f;
        a.video[k] = (unsigned char)g;
        a.tmp_off[k] = need;
        a.first_block[k] = (int)blocks;
        need += (long long)f.Hc * res * 3;
        blocks += ceil_div((long long)f.Hc * res, 256);
    }
    if (tmp_floats < need) return DBOA_ERR_ARG;
    if (blocks > 0x7fffffffLL) return DBOA_ERR_SHAPE;
    a.first_block[a.n] = (int)blocks;
    for (int c = 0; c < 3; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
    crop_groups_rows_kernel<<<(unsigned)blocks, 256, 0, st>>>(a, tmp);
    DBOA_TRY(check_launch());
    crop_groups_cols_kernel<<<dim3(ceil_div((long long)res * res, 256), a.n), 256, 0, st>>>(a, tmp, out);
    return check_launch();
}

// one frame: the grouped call with a single descriptor
int crop_resize_normalize(const void* img, int is_u8, int H, int W, int ul_x, int ul_y, int Hc, const float* wx, const int* sx, int Tx,
                          const float* wy, const int* sy, int Ty, int res, const float mean[3], const float stdv[3], float* tmp, float* out,
                          cudaStream_t st) {
    if (H < 1 || W < 1 || Hc < 1 || Tx < 1 || Ty < 1 || res < 1) return DBOA_ERR_SHAPE;
    dboa_crop_desc d;
    d.img = img; d.wx = wx; d.sx = sx; d.wy = wy; d.sy = sy;
    d.is_u8 = is_u8; d.H = H; d.W = W; d.ul_x = ul_x; d.ul_y = ul_y; d.Hc = Hc; d.Tx = Tx; d.Ty = Ty;
    return crop_resize_normalize_groups(&d, 1, 1ULL, res, mean, stdv, tmp, (long long)Hc * res * 3, out, st);
}

struct KeypointGroups {
    double t[64][4];              // entry k: t00, t02, t11, t12 of video video[k]
    unsigned char video[64];
    int n, res;
};
// block k: rows [0, 49) of entry k's video; rows >= n are zeroed
__global__ void __launch_bounds__(64) keypoint_groups_kernel(const __grid_constant__ KeypointGroups a, const float* __restrict__ kp,
                                                             float* __restrict__ out) {
    const int k = blockIdx.x, j = threadIdx.x, g = a.video[k];
    if (j >= 49) return;
    float* o = out + ((size_t)g * 49 + j) * 3;
    if (j >= a.n) {
        o[0] = 0.f; o[1] = 0.f; o[2] = 0.f;
        return;
    }
    keypoint_elem(kp + ((size_t)g * a.n + j) * 3, a.t[k][0], a.t[k][1], a.t[k][2], a.t[k][3], a.res, o);
}
int keypoint_transform_groups(const float* kp, int n, const double* t4, int res, float* out, int groups, unsigned long long active,
                              cudaStream_t st) {
    if (groups < 1 || groups > 64 || n < 0 || n > 49 || res < 1) return DBOA_ERR_SHAPE;
    if (!mask_ok(groups, active)) return DBOA_ERR_ARG;
    KeypointGroups a;
    a.n = n; a.res = res;
    int m = 0;
    for (int g = 0; g < groups; ++g) {
        if (!((active >> g) & 1ULL)) continue;
        for (int c = 0; c < 4; ++c) a.t[m][c] = t4[g * 4 + c];
        a.video[m++] = (unsigned char)g;
    }
    keypoint_groups_kernel<<<m, 64, 0, st>>>(a, kp, out);
    return check_launch();
}

}  // namespace dboa
