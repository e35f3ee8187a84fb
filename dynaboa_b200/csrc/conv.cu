// fp32 implicit-GEMM convolution on CUDA cores: forward, data gradient, weight gradient.
//
// Replaces the cuDNN calls behind reference model/hmr.py:29-34,72,113 (53 x nn.Conv2d, bias=False)
// and their autograd backward (SURVEY.md §2.1 K1).  Activations are NHWC; weights are
// [Cout][kh][kw][Cin] with a row pitch `Kpitch >= roundup16(kh*kw*Cin)` (zero padded).
//
// This is the exact-fp32 path: it is the numerical reference the wgmma TF32x3 path
// (conv_tc.cu) is checked against on the GPU, and it serves the shapes that path does not
// take (Cin = 3 stem, odd tiles).  Split-K is deterministic: the K slices of a tile form a cluster
// whose partial tiles are summed in a fixed order through distributed shared memory (cluster_reduce_store).
#include <cooperative_groups.h>

#include "common.cuh"
#include "kernels.h"

namespace cg = cooperative_groups;

namespace dboa {

constexpr int BM = 64, BN = 64, BK = 16, NT = 256, PADM = 4;
constexpr int PF = 4;      // slabs of operand loads kept in flight per thread

// One BK-deep slab of the 64x64 tile product; thread (tx,ty) owns a 4x4 micro-tile.
__device__ __forceinline__ void mma_slab(const float (*As)[BM + PADM], const float (*Bs)[BN + PADM], int tx, int ty,
                                         float acc[4][4]) {
#pragma unroll
    for (int k = 0; k < BK; ++k) {
        float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
}

// Split-K across a thread-block cluster (cluster dims (1,1,nz), nz <= 8): every K-slice parks its 64x64 partial
// tile in its own shared memory, the cluster synchronises in hardware, and each CTA then sums a band of 64/nz rows over
// all peers through distributed shared memory in the fixed order z = 0..nz-1 (deterministic) and writes that band.
// No global partials, no atomics, no second launch.  `ncols` bounds the columns (weight gradient of the 7x7 stem).
__device__ __forceinline__ void cluster_reduce_store(const float acc[4][4], float* red, float* __restrict__ out, int nrows, int ld,
                                                     int r0, int c0, int ncols, int tx, int ty, int accumulate) {
    const int nz = gridDim.z;
    if (nz == 1) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int row = r0 + ty * 4 + i;
            if (row >= nrows) continue;
            float* p = out + (size_t)row * ld + c0 + tx * 4;
            if (c0 + tx * 4 + 3 < ncols) {
                float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
                if (accumulate) { float4 c = *reinterpret_cast<float4*>(p); v.x += c.x; v.y += c.y; v.z += c.z; v.w += c.w; }
                *reinterpret_cast<float4*>(p) = v;
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (c0 + tx * 4 + j < ncols) p[j] = accumulate ? p[j] + acc[i][j] : acc[i][j];
            }
        }
        return;
    }
    cg::cluster_group cluster = cg::this_cluster();
#pragma unroll
    for (int i = 0; i < 4; ++i)
        *reinterpret_cast<float4*>(red + (ty * 4 + i) * BN + tx * 4) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    cluster.sync();
    const int rank = (int)cluster.block_rank();
    const int rows_per = BM / nz;                         // nz is a power of two <= 16
    for (int v = threadIdx.x; v < rows_per * (BN / 4); v += NT) {
        const int lr = rank * rows_per + v / (BN / 4), c4 = (v % (BN / 4)) * 4;
        const int row = r0 + lr;
        if (row >= nrows) continue;
        float4 q[16];                                     // all remote loads in flight before the first add (DSMEM latency ~200 cycles each)
#pragma unroll
        for (int z = 0; z < 16; ++z)
            if (z < nz) q[z] = *reinterpret_cast<const float4*>(cluster.map_shared_rank(red, z) + lr * BN + c4);
        float4 sacc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int z = 0; z < 16; ++z)
            if (z < nz) { sacc.x += q[z].x; sacc.y += q[z].y; sacc.z += q[z].z; sacc.w += q[z].w; }
        float* p = out + (size_t)row * ld + c0 + c4;
        if (c0 + c4 + 3 < ncols) {
            if (accumulate) { float4 c = *reinterpret_cast<float4*>(p); sacc.x += c.x; sacc.y += c.y; sacc.z += c.z; sacc.w += c.w; }
            *reinterpret_cast<float4*>(p) = sacc;
        } else {
            const float sv[4] = {sacc.x, sacc.y, sacc.z, sacc.w};
            for (int j = 0; j < 4; ++j)
                if (c0 + c4 + j < ncols) p[j] = accumulate ? p[j] + sv[j] : sv[j];
        }
    }
    cluster.sync();                                        // peers may still be reading this CTA's tile
}

// ---------------------------------------------------------------------------------------------
// forward:  y[m][n] = sum_k xcol[m][k] * w[n][k],   m = (b,ho,wo), k = (r,s,ci)
// grid (ceil(M/64), Cout/64, nsplit); each z-slice covers k in [z*klen, (z+1)*klen)
// ---------------------------------------------------------------------------------------------
// GROUPED (all three kernels): a call over d.groups > 1 groups; the group arithmetic is compiled only into that instantiation.
// The CTAs of an idle group (d.active bit clear) return before the cluster reduction, so a split-K cluster (along z, inside one
// group) exits as a whole.
template <int VEC, bool GROUPED>
__global__ void __launch_bounds__(NT) conv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                      float* __restrict__ out, ConvDims d, int klen) {
    __shared__ __align__(16) float As[BK][BM + PADM];
    __shared__ __align__(16) float Bs[BK][BN + PADM];
    __shared__ __align__(16) float red[BM * BN];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int M = d.B * d.Ho * d.Wo, K = d.kh * d.kw * d.Cin;
    int bx = blockIdx.x;
    if (GROUPED) {                                                       // the row tiles of group grp
        const int gx = gridDim.x / d.groups, grp = blockIdx.x / gx;
        if (!((d.active >> grp) & 1ULL)) return;
        x +=(size_t)grp * d.B * d.Hi * d.Wi * d.Cin; w += grp * d.wstride; out += (size_t)grp * M * d.Cout;
        bx -= grp * gx;
    }
    const int m0 = bx * BM, n0 = blockIdx.y * BN;
    const int kbeg = blockIdx.z * klen, kend = min(kbeg + klen, (K + BK - 1) / BK * BK);

    // loader roles: row = tid/4, kv = tid%4 (4 consecutive k)
    const int lrow = tid >> 2, lkv = (tid & 3) * 4;
    const int m = m0 + lrow;
    const bool mvalid = m < M;
    int hi0 = 0, wi0 = 0;
    const float* xb = x;
    if (mvalid) {
        int b = m / (d.Ho * d.Wo), rem = m - b * d.Ho * d.Wo;
        int ho = rem / d.Wo, wo = rem - ho * d.Wo;
        hi0 = ho * d.stride - d.pad; wi0 = wo * d.stride - d.pad;
        xb = x + (size_t)b * d.Hi * d.Wi * d.Cin;
    }
    const float* wrow = w + (size_t)(n0 + lrow) * d.Kpitch;

    // operand fetch for the k-slab starting at k0 (registers; issued one slab ahead of the math)
    auto fetch = [&](int k0, float (&av)[4], float4& bv) {
        const int k = k0 + lkv;
        av[0] = av[1] = av[2] = av[3] = 0.f;
        if (mvalid) {
            if (VEC == 4) {
                if (k < K) {
                    int tap = k / d.Cin, ci = k - tap * d.Cin;
                    int r = tap / d.kw, s = tap - r * d.kw;
                    int hi = hi0 + r, wi = wi0 + s;
                    if ((unsigned)hi < (unsigned)d.Hi && (unsigned)wi < (unsigned)d.Wi) {
                        float4 v = ldg4(xb + ((size_t)hi * d.Wi + wi) * d.Cin + ci);
                        av[0] = v.x; av[1] = v.y; av[2] = v.z; av[3] = v.w;
                    }
                }
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    int kk = k + e;
                    if (kk < K) {
                        int tap = kk / d.Cin, ci = kk - tap * d.Cin;
                        int r = tap / d.kw, s = tap - r * d.kw;
                        int hi = hi0 + r, wi = wi0 + s;
                        if ((unsigned)hi < (unsigned)d.Hi && (unsigned)wi < (unsigned)d.Wi)
                            av[e] = __ldg(xb + ((size_t)hi * d.Wi + wi) * d.Cin + ci);
                    }
                }
            }
        }
        bv = ldg4(wrow + k);                  // rows are zero padded up to Kpitch >= roundup16(K)
    };
    // register pipeline, PF slabs deep: at batch 1 the weight-streaming layers are bound by memory latency per CTA,
    // so several slabs of loads stay in flight while one slab is multiplied 
    float acc[4][4] = {};
    float av[PF][4];
    float4 bv[PF];
    pdl_wait();                             // index set-up above overlaps the previous kernel's tail
    pdl_trigger();
#pragma unroll
    for (int f = 0; f < PF; ++f)
        if (kbeg + f * BK < kend) fetch(kbeg + f * BK, av[f], bv[f]);
    for (int k0 = kbeg; k0 < kend; k0 += PF * BK) {
#pragma unroll
        for (int f = 0; f < PF; ++f) {
            const int kk = k0 + f * BK;
            if (kk < kend) {
                __syncthreads();
                As[lkv + 0][lrow] = av[f][0]; As[lkv + 1][lrow] = av[f][1]; As[lkv + 2][lrow] = av[f][2]; As[lkv + 3][lrow] = av[f][3];
                Bs[lkv + 0][lrow] = bv[f].x; Bs[lkv + 1][lrow] = bv[f].y; Bs[lkv + 2][lrow] = bv[f].z; Bs[lkv + 3][lrow] = bv[f].w;
                __syncthreads();
                if (kk + PF * BK < kend) fetch(kk + PF * BK, av[f], bv[f]);
                mma_slab(As, Bs, tx, ty, acc);
            }
        }
    }
    cluster_reduce_store(acc, red, out, M, d.Cout, m0, n0, d.Cout, tx, ty, 0);
}

// ---------------------------------------------------------------------------------------------
// data gradient:  dx[m][ci] = sum_{r,s,co} dy[b][ho][wo][co] * w[co][r][s][ci]
//   m = (b,hi,wi);  ho = (hi + pad - r)/stride when divisible and in range
// GEMM view: M = B*Hi*Wi, N = Cin, K = kh*kw*Cout ordered (r,s,co)
// ---------------------------------------------------------------------------------------------
template <bool GROUPED>
__global__ void __launch_bounds__(NT) conv_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w,
                                                        float* __restrict__ out, ConvDims d, int klen, int accumulate) {
    __shared__ __align__(16) float As[BK][BM + PADM];
    __shared__ __align__(16) float Bs[BK][BN + PADM];
    __shared__ __align__(16) float red[BM * BN];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int M = d.B * d.Hi * d.Wi, K = d.kh * d.kw * d.Cout;
    int bx = blockIdx.x;
    if (GROUPED) {
        const int gx = gridDim.x / d.groups, grp = blockIdx.x / gx;
        if (!((d.active >> grp) & 1ULL)) return;
        dy += (size_t)grp * d.B * d.Ho * d.Wo * d.Cout; w += grp * d.wstride; out += (size_t)grp * M * d.Cin;
        bx -= grp * gx;
    }
    const int m0 = bx * BM, n0 = blockIdx.y * BN;
    const int kbeg = blockIdx.z * klen, kend = min(kbeg + klen, K);

    const int lrow = tid >> 2, lkv = (tid & 3) * 4;       // A loader: 4 consecutive co
    const int m = m0 + lrow;
    const bool mvalid = m < M;
    int hi = 0, wi = 0;
    const float* dyb = dy;
    if (mvalid) {
        int b = m / (d.Hi * d.Wi), rem = m - b * d.Hi * d.Wi;
        hi = rem / d.Wi; wi = rem - hi * d.Wi;
        dyb = dy + (size_t)b * d.Ho * d.Wo * d.Cout;
    }
    const int bk = tid >> 4, bnv = (tid & 15) * 4;        // B loader: row k, 4 consecutive ci

    auto fetch = [&](int k0, float4& av, float4& bv) {
        av = make_float4(0.f, 0.f, 0.f, 0.f);
        bv = make_float4(0.f, 0.f, 0.f, 0.f);
        {
            const int k = k0 + lkv;
            if (mvalid && k < kend) {
                int tap = k / d.Cout, co = k - tap * d.Cout;
                int r = tap / d.kw, s = tap - r * d.kw;
                int th = hi + d.pad - r, tw = wi + d.pad - s;
                if (th >= 0 && tw >= 0) {
                    int ho = th / d.stride, wo = tw / d.stride;
                    if (ho * d.stride == th && wo * d.stride == tw && ho < d.Ho && wo < d.Wo)
                        av = ldg4(dyb + ((size_t)ho * d.Wo + wo) * d.Cout + co);
                }
            }
        }
        {
            const int k = k0 + bk;
            if (k < kend) {
                int tap = k / d.Cout, co = k - tap * d.Cout;
                bv = ldg4(w + (size_t)co * d.Kpitch + (size_t)tap * d.Cin + n0 + bnv);
            }
        }
    };
    float acc[4][4] = {};
    float4 av[PF], bv[PF];
    pdl_wait();                             // index set-up above overlaps the previous kernel's tail
    pdl_trigger();
#pragma unroll
    for (int f = 0; f < PF; ++f)
        if (kbeg + f * BK < kend) fetch(kbeg + f * BK, av[f], bv[f]);
    for (int k0 = kbeg; k0 < kend; k0 += PF * BK) {
#pragma unroll
        for (int f = 0; f < PF; ++f) {
            const int kk = k0 + f * BK;
            if (kk < kend) {
                __syncthreads();
                As[lkv + 0][lrow] = av[f].x; As[lkv + 1][lrow] = av[f].y; As[lkv + 2][lrow] = av[f].z; As[lkv + 3][lrow] = av[f].w;
                *reinterpret_cast<float4*>(&Bs[bk][bnv]) = bv[f];
                __syncthreads();
                if (kk + PF * BK < kend) fetch(kk + PF * BK, av[f], bv[f]);
                mma_slab(As, Bs, tx, ty, acc);
            }
        }
    }
    cluster_reduce_store(acc, red, out, M, d.Cin, m0, n0, d.Cin, tx, ty, accumulate);
}

// ---------------------------------------------------------------------------------------------
// weight gradient:  dw[co][(r,s,ci)] (+)= sum_m dy[m][co] * xcol[m][(r,s,ci)]
// GEMM view: M' = Cout, N' = kh*kw*Cin, K' = B*Ho*Wo (split over blockIdx.z)
// ---------------------------------------------------------------------------------------------
template <int VEC, bool GROUPED>
__global__ void __launch_bounds__(NT) conv_wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                        float* __restrict__ out, ConvDims d, int plen) {
    __shared__ __align__(16) float As[BK][BM + PADM];
    __shared__ __align__(16) float Bs[BK][BN + PADM];
    __shared__ __align__(16) float red[BM * BN];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int Mpix = d.B * d.Ho * d.Wo, K = d.kh * d.kw * d.Cin;
    int bx = blockIdx.x;
    if (GROUPED) {                                                       // K' = this group's B*Ho*Wo pixels
        const int gx = gridDim.x / d.groups, grp = blockIdx.x / gx;
        if (!((d.active >> grp) & 1ULL)) return;
        dy += (size_t)grp * Mpix * d.Cout; x += (size_t)grp * d.B * d.Hi * d.Wi * d.Cin; out += grp * d.wstride;
        bx -= grp * gx;
    }
    const int m0 = bx * BM /* co */, n0 = blockIdx.y * BN /* (r,s,ci) */;
    const int pbeg = blockIdx.z * plen, pend = min(pbeg + plen, Mpix);

    const int lk = tid >> 4, lv = (tid & 15) * 4;
    // B loader: this thread's 4 columns n' = n0 + lv .. +3
    int br[4], bs[4], bc[4]; bool bval[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        int n = n0 + lv + e;
        bval[e] = n < K;
        int tap = bval[e] ? n / d.Cin : 0;
        bc[e] = bval[e] ? n - tap * d.Cin : 0;
        br[e] = tap / d.kw; bs[e] = tap - br[e] * d.kw;
    }

    auto fetch = [&](int p0, float4& av, float (&bv)[4]) {
        const int p = p0 + lk;
        av = make_float4(0.f, 0.f, 0.f, 0.f);
        bv[0] = bv[1] = bv[2] = bv[3] = 0.f;
        if (p < pend) {
            av = ldg4(dy + (size_t)p * d.Cout + m0 + lv);
            int b = p / (d.Ho * d.Wo), rem = p - b * d.Ho * d.Wo;
            int ho = rem / d.Wo, wo = rem - ho * d.Wo;
            const float* xb = x + (size_t)b * d.Hi * d.Wi * d.Cin;
            if (VEC == 4) {
                if (bval[0]) {
                    int hi = ho * d.stride - d.pad + br[0], wi = wo * d.stride - d.pad + bs[0];
                    if ((unsigned)hi < (unsigned)d.Hi && (unsigned)wi < (unsigned)d.Wi) {
                        float4 v = ldg4(xb + ((size_t)hi * d.Wi + wi) * d.Cin + bc[0]);
                        bv[0] = v.x; bv[1] = v.y; bv[2] = v.z; bv[3] = v.w;
                    }
                }
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (bval[e]) {
                        int hi = ho * d.stride - d.pad + br[e], wi = wo * d.stride - d.pad + bs[e];
                        if ((unsigned)hi < (unsigned)d.Hi && (unsigned)wi < (unsigned)d.Wi)
                            bv[e] = __ldg(xb + ((size_t)hi * d.Wi + wi) * d.Cin + bc[e]);
                    }
            }
        }
    };
    float acc[4][4] = {};
    float4 av[PF];
    float bv[PF][4];
    pdl_wait();                             // index set-up above overlaps the previous kernel's tail
    pdl_trigger();
#pragma unroll
    for (int f = 0; f < PF; ++f)
        if (pbeg + f * BK < pend) fetch(pbeg + f * BK, av[f], bv[f]);
    for (int p0 = pbeg; p0 < pend; p0 += PF * BK) {
#pragma unroll
        for (int f = 0; f < PF; ++f) {
            const int pp = p0 + f * BK;
            if (pp < pend) {
                __syncthreads();
                *reinterpret_cast<float4*>(&As[lk][lv]) = av[f];
                *reinterpret_cast<float4*>(&Bs[lk][lv]) = make_float4(bv[f][0], bv[f][1], bv[f][2], bv[f][3]);
                __syncthreads();
                if (pp + PF * BK < pend) fetch(pp + PF * BK, av[f], bv[f]);
                mma_slab(As, Bs, tx, ty, acc);
            }
        }
    }
    // rows = co, cols = n'; the weight gradient always accumulates (+=) into the gradient arena
    cluster_reduce_store(acc, red, out, d.Cout, d.Kpitch, m0, n0, K, tx, ty, 1);
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
// K-slices per tile: a power of two <= 8 (the portable cluster size) that fills ~2 waves and leaves >= 4 iterations
static int pick_split(int tiles, int kiters) {
    const int target = 2 * num_sms();
    int ns = 1;
    while (ns < 8 && tiles * ns * 2 <= target + tiles && kiters / (ns * 2) >= 4) ns *= 2;
    return ns;
}

template <typename K, typename... Args>
static int launch_z_cluster(K kernel, dim3 grid, cudaStream_t st, Args... args) {
    return launch_ex(kernel, grid, dim3(NT), 0, st, dim3(1, 1, grid.z), true, args...);
}

int conv_fwd(const float* x, const float* w, float* y, const ConvDims& d, float* ws, size_t ws_floats, cudaStream_t st) {
    (void)ws; (void)ws_floats;
    if (d.groups < 1) return DBOA_ERR_SHAPE;
    if (d.Cout % BN != 0 || d.Kpitch % 4 != 0) return DBOA_ERR_SHAPE;
    const int M = d.B * d.Ho * d.Wo, K = d.kh * d.kw * d.Cin;
    if (d.Kpitch < (K + BK - 1) / BK * BK) return DBOA_ERR_SHAPE;
    const int kiters = (K + BK - 1) / BK;
    const int tiles = d.groups * ceil_div(M, BM) * (d.Cout / BN);
    const int ns = pick_split(tiles, kiters);
    const int klen = ((kiters + ns - 1) / ns) * BK;
    dim3 grid(d.groups * ceil_div(M, BM), d.Cout / BN, ns);
    const bool g = d.groups > 1;
    if (d.Cin % 4 == 0) return launch_z_cluster(g ? conv_fwd_kernel<4, true> : conv_fwd_kernel<4, false>, grid, st, x, w, y, d, klen);
    return launch_z_cluster(g ? conv_fwd_kernel<1, true> : conv_fwd_kernel<1, false>, grid, st, x, w, y, d, klen);
}

int conv_dgrad(const float* dy, const float* w, float* dx, const ConvDims& d, int accumulate, float* ws, size_t ws_floats,
               cudaStream_t st) {
    (void)ws; (void)ws_floats;
    if (d.groups < 1) return DBOA_ERR_SHAPE;
    if (d.Cin % BN != 0 || d.Cout % BK != 0) return DBOA_ERR_SHAPE;
    const int M = d.B * d.Hi * d.Wi, K = d.kh * d.kw * d.Cout;
    const int kiters = K / BK;
    const int tiles = d.groups * ceil_div(M, BM) * (d.Cin / BN);
    const int ns = pick_split(tiles, kiters);
    const int klen = ((kiters + ns - 1) / ns) * BK;
    dim3 grid(d.groups * ceil_div(M, BM), d.Cin / BN, ns);
    return launch_z_cluster(d.groups > 1 ? conv_dgrad_kernel<true> : conv_dgrad_kernel<false>, grid, st, dy, w, dx, d, klen, accumulate);
}

int conv_wgrad(const float* dy, const float* x, float* dw, const ConvDims& d, float* ws, size_t ws_floats, cudaStream_t st) {
    // the stem has its own kernel (last on the critical path of every backward); the generic kernel below takes every other shape
    const int s = stem_wgrad(dy, x, dw, d, ws, ws_floats, st);
    if (s != DBOA_ERR_UNSUPPORTED) return s;
    if (d.Cout % BM != 0 || d.groups < 1) return DBOA_ERR_SHAPE;
    const int Mpix = d.B * d.Ho * d.Wo, K = d.kh * d.kw * d.Cin;
    const int piters = ceil_div(Mpix, BK);
    const int tiles = d.groups * (d.Cout / BM) * ceil_div(K, BN);
    const int ns = pick_split(tiles, piters);
    const int plen = ((piters + ns - 1) / ns) * BK;
    dim3 grid(d.groups * (d.Cout / BM), ceil_div(K, BN), ns);
    const bool g = d.groups > 1;
    if (d.Cin % 4 == 0) return launch_z_cluster(g ? conv_wgrad_kernel<4, true> : conv_wgrad_kernel<4, false>, grid, st, dy, x, dw, d, plen);
    return launch_z_cluster(g ? conv_wgrad_kernel<1, true> : conv_wgrad_kernel<1, false>, grid, st, dy, x, dw, d, plen);
}

}  // namespace dboa
