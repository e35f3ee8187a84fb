// wgmma (Hopper warpgroup tensor core) implicit-GEMM convolution: forward, data gradient and weight gradient of
// every backbone convolution with Cin % 64 == 0 and Cout % 64 == 0 (all but the 7x7 stem).
//
//   FWD   : Y [m=(b,ho,wo)][n=co]      = sum_{k=(tap,ci)} Xcol[m][k]  * W[co][k]
//   DGRAD : dX[m=(b,hi,wi)][n=ci]   (+)= sum_{k=(tap,co)} dYcol[m][k] * W[co][tap][ci]
//   WGRAD : dW[m=co][n=(tap,ci)]      += sum_{k=pixel}    dY[pix][co] * Xcol[pix][(tap,ci)]
// activations NHWC, weights [Cout][kh][kw][Cin] (row pitch == kh*kw*Cin).
//
// Precision: `wgmma.mma_async ... .tf32.tf32` with a 3-term split.  Every operand value x is split by the loader threads
// into hi = x with the low 13 mantissa bits cleared (exactly a TF32 number, so the tensor core's own fp32->tf32
// conversion is the identity) and lo = x - hi (exact in fp32); the accumulator receives
//   Ah*Bh + Ah*Bl + Al*Bh      (the dropped Al*Bl term is ~2^-22 relative)
// The tensor core adds into its fp32 accumulator with truncation, so a long chain of accumulations drifts towards zero
// (~n * 2^-25 relative after n additions); each k-block therefore starts a fresh accumulator of 12 products, which is added
// to the running fp32 total in registers with round-to-nearest.  The result stays within ~2e-6 of the exact-fp32 CUDA-core path (conv.cu), against
// which this kernel is validated on the device (tests/test_gpu_tc.py).  SURVEY.md §7 "hard part 1".
//
// Structure (one CTA = 2 warpgroups = 256 threads, one 128 x 64 output tile, 32 reduction elements per k-block):
//   loaders  : every thread loads per k-block 2 float4 of the 128-row operand and 1 of the 64-row operand; im2col /
//              transposed-filter / pixel-major gathers computed on the fly with zero fill, issued two k-blocks ahead
//              in registers; a warp request covers 8 rows x 64 contiguous bytes.  hi/lo are split in registers and
//              stored into the canonical K-major no-swizzle layout (8-row x 16-byte core matrices) of one of 2
//              shared-memory stages.  Operands whose memory order is reduction-minor (K-major) are stored with float4
//              (conflict free); the others are transposed by the store.
//   MMA      : warpgroup g issues 12 x wgmma m64n64k8 (4 k-steps of {Ah*Bh, Ah*Bl, Al*Bh}) on rows 64g .. 64g + 63 of
//              the filled stage; the global loads of a later k-block are issued before the wait, so they are in flight
//              while the MMAs run.  Per thread 32 fp32 registers of the k-block's accumulator and 32 of the running total.
//   epilogue : registers -> shared memory -> row-contiguous global stores.  Split-K runs across a thread-block cluster
//              (1,1,nz): each CTA sums a band of 128/nz rows over its peers through distributed shared memory (all remote
//              loads in flight, then added in the fixed order z = 0..nz-1).
#include <cooperative_groups.h>
#include <stdint.h>
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"

namespace cg = cooperative_groups;

namespace dboa {

// 0 = fp32 CUDA cores; 1 = forward on tensor cores; 2 = forward, data and weight gradient on tensor cores;
// 3 = forward and data gradient on tensor cores, weight gradient on CUDA cores (default: C2 at batch 1 on an H100 SXM, 700 W,
// runs alternated in one session: 129.0-129.1 adapted frames/s against 116.3-116.6 with mode 2; a batch-1 weight gradient
// reduces over few pixels into many outputs, which the CUDA-core kernel's cluster split serves better)
static int g_tc_mode = 3;
bool conv_tc_enabled() { return g_tc_mode != 0; }
bool conv_tc_bwd_enabled() { return g_tc_mode >= 2; }
bool conv_tc_wgrad_enabled() { return g_tc_mode == 2; }
void conv_tc_set_enabled(bool on) { g_tc_mode = on ? 2 : 0; }
void conv_tc_set_mode(int mode) { g_tc_mode = mode; }

namespace tc {

// Diagnostic build (-DDBOA_TIMELINE, buffer set by dboa_debug_set_timeline): thread 0 of every CTA stamps %globaltimer at the phase
// boundaries of the kernel into a device buffer [cta][16]; compiled out of the product library.
#ifdef DBOA_TIMELINE
__device__ unsigned long long* g_timeline = nullptr;
#define DBOA_TL(i)                                                                                        \
    do {                                                                                                  \
        if (threadIdx.x == 0 && g_timeline != nullptr) {                                                  \
            unsigned long long t_;                                                                        \
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));                                        \
            g_timeline[((size_t)(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * 16 + (i)] = t_; \
        }                                                                                                 \
    } while (0)
// per-iteration cycle stamps of CTA (0,0,0), thread 0: slot 40000 + it * 8 + j
#define DBOA_TLC(it, j)                                                                                   \
    do {                                                                                                  \
        if (threadIdx.x == 0 && g_timeline != nullptr && (blockIdx.x | blockIdx.y | blockIdx.z) == 0 && (it) < 12)   \
            g_timeline[40000 + (it) * 8 + (j)] = (unsigned long long)clock64();                           \
    } while (0)
#else
#define DBOA_TL(i)
#define DBOA_TLC(it, j)
#endif

enum { FWD = 0, DGRAD = 1, WGRAD = 2 };
constexpr int BM = 128, BN = 64, BK = 32, STAGES = 2;
constexpr int NPW = 8, NPROD = NPW * 32, NT = NPROD;          // 8 loader warps = the 2 MMA warpgroups
constexpr uint32_t CORE_BYTES = 128;                     // one 8 x 16B core matrix
constexpr uint32_t GROUP_BYTES = (BK / 4) * CORE_BYTES;  // one 8-row group of a stage tile (1024 B)
constexpr uint32_t A_TILE = BM * BK * 4, B_TILE = BN * BK * 4;
constexpr int RED_LD = BN + 4;                           // padded row pitch of the split-K partial tile (bank-conflict free)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    // wgmma shared-memory matrix descriptor: start[0,14) | LBO[16,30) | SBO[32,46) | layout_type[62,64) = 0 (no swizzle), in 16-byte units.
    // K-major: LBO = byte step between the two 16-byte k-chunks of one MMA, SBO = byte step between 8-row groups
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((CORE_BYTES >> 4) & 0x3FFF) << 16) |
           ((uint64_t)((GROUP_BYTES >> 4) & 0x3FFF) << 32);
}

// d[64 x 64] += A[64 x 8] * B[64 x 8]^T (both K-major in shared memory), issued by the whole warpgroup.  Accumulator fragment:
// d[i] is row 16 * (warp % 4) + lane / 4 + 8 * ((i >> 1) & 1), column 8 * (i >> 2) + 2 * (lane % 4) + (i & 1).
// scale_d == 0: d = A * B^T (the accumulator's previous contents are ignored)
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc, int scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(scale_d)
        : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Pins the accumulator registers at the fences of the asynchronous region (CUTLASS warpgroup_fence_operand): without it the
// compiler may move ordinary register writes into the region and then serialises every wgmma (ptxas C7515).
__device__ __forceinline__ void fence_operand(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i]));
}

__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// K-major source: 4 consecutive reduction elements of one row -> one float4 slot of the canonical layout
__device__ __forceinline__ void split_store4(uint8_t* hi_tile, uint8_t* lo_tile, uint32_t off, float4 v) {
    float4 h = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
    *reinterpret_cast<float4*>(hi_tile + off) = h;
    *reinterpret_cast<float4*>(lo_tile + off) = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
}
// row-minor source: 4 consecutive ROWS (row0 % 4 == 0) at one reduction index k -> 4 scalar slots (transposing store)
__device__ __forceinline__ void split_store_t(uint8_t* hi_tile, uint8_t* lo_tile, int row0, int k, float4 v) {
    const uint32_t off = (uint32_t)(row0 >> 3) * GROUP_BYTES + (uint32_t)(k >> 2) * CORE_BYTES + (uint32_t)(row0 & 7) * 16 + (uint32_t)(k & 3) * 4;
    const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float h = tf32_hi(x[e]);
        *reinterpret_cast<float*>(hi_tile + off + e * 16) = h;
        *reinterpret_cast<float*>(lo_tile + off + e * 16) = x[e] - h;
    }
}

// same, with the 4 element stores issued in the order (e + rot) & 3: when the lanes of a warp are (k & 3, (row0 >> 2) & 1, rot)
// the 32 scalar stores of one instruction fall into 32 different banks (the plain version is an 8-way conflict)
__device__ __forceinline__ void split_store_t_rot(uint8_t* hi_tile, uint8_t* lo_tile, int row0, int k, float4 v, int rot) {
    const uint32_t off = (uint32_t)(row0 >> 3) * GROUP_BYTES + (uint32_t)(k >> 2) * CORE_BYTES + (uint32_t)(row0 & 7) * 16 + (uint32_t)(k & 3) * 4;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int ee = (e + rot) & 3;
        const float x = ee == 0 ? v.x : (ee == 1 ? v.y : (ee == 2 ? v.z : v.w));
        const float h = tf32_hi(x);
        *reinterpret_cast<float*>(hi_tile + off + ee * 16) = h;
        *reinterpret_cast<float*>(lo_tile + off + ee * 16) = x - h;
    }
}

struct Smem {
    // stage tiles in the canonical K-major layout: [row_group][k_chunk][8 rows][16 B]; after the last MMA the A tiles are
    // re-used as the 128 x RED_LD fp32 tile of the epilogue
    alignas(128) uint8_t a_hi[STAGES][A_TILE];
    alignas(128) uint8_t a_lo[STAGES][A_TILE];
    alignas(128) uint8_t b_hi[STAGES][B_TILE];
    alignas(128) uint8_t b_lo[STAGES][B_TILE];
    float2 gn[2][256];     // fused variants: per (sample, group) operand GroupNorm (mean, rstd); data gradient: (mean, rstd), (m1, m2)
};

// Operand transforms and epilogue sums of the fused variants (XF: -1 none; 0..3 forward, kernels.h FusedConv::mode; XD data
// gradient, kernels.h DgradFused).  Fixed-point scales: 2^24 for forward statistics, 2^28 for backward sums.
constexpr int XD = 10;
struct Ext {
    const float* res; const long long *acc_in, *acc2_in; const float *gamma, *beta, *gamma2, *beta2;
    float *a_out, *stats_out, *stats2_out; long long* acc_out;
    const float *y_c, *stats_c; const long long* sums_c; const float* gamma_c; float* dy_out; const float *addend, *mask;
    const float* prep_y[2]; const float* prep_stats[2]; const float* prep_gamma[2]; long long* prep_sums[2]; long long* prep_dgb[2];
    int nprep;
};
constexpr double FIX_FWD = 16777216.0, FIX_BWD = 268435456.0;
__device__ __forceinline__ void add_fixed(long long* p, double v, double scale) {
    atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)llrint(v * scale));
}

// P: the operand that pairs with the weights in FWD/DGRAD (x or dy); Q: weights (FWD/DGRAD) or x (WGRAD, with P = dy)
// GROUPED: a call over d.groups > 1 groups (the group arithmetic is compiled only into this instantiation)
template <int MODE, int XF, bool GROUPED = false>
__global__ void __launch_bounds__(NT, 1) conv_tf32x3_kernel(const float* __restrict__ P, const float* __restrict__ Q, float* __restrict__ O,
                                                            ConvDims d, int kb_per_split, int accumulate, const Ext e) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
    float2 (&s_gn)[2][256] = sm.gn;
    constexpr bool XFWD = XF >= 1 && XF <= 3, XDG = XF == XD, XOP = XFWD || XDG;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    DBOA_TL(0);
    const int Ktaps = d.kh * d.kw, Kfull = Ktaps * d.Cin;
    // Grouped call: blockIdx.x = group * gx + tile, and group grp reads / writes only its own samples and weights (no tile
    // straddles two groups, since the weight operand differs per group).  groups == 1: grp = 0, bx = blockIdx.x.
    // The CTAs of an idle group (its `d.active` bit clear) return here: the split-K cluster lies along z inside one group, so the
    // exit is uniform over the cluster and comes before any barrier, DSMEM access or dependency wait.
    int gx = gridDim.x, bx = blockIdx.x;
    if (GROUPED) {
        const int grp = blockIdx.x / (gridDim.x / d.groups);
        if (!((d.active >> grp) & 1ULL)) return;
        gx = gridDim.x / d.groups; bx = blockIdx.x - grp * gx;
        const size_t xin = (size_t)grp * d.B * d.Hi * d.Wi * d.Cin, yout = (size_t)grp * d.B * d.Ho * d.Wo * d.Cout;
        if (MODE == FWD) { P += xin; Q += grp * d.wstride; O += yout; }
        else if (MODE == DGRAD) { P += yout; Q += grp * d.wstride; O += xin; }
        else { P += yout; Q += xin; O += grp * d.wstride; }
    }
    // GEMM extents of this mode
    // Stride-2 data gradient: an input pixel (hi, wi) only receives the filter taps r = hi + pad (mod 2), s = wi + pad (mod 2).
    // The rows are therefore enumerated per PARITY CLASS (hi & 1, wi & 1): blockIdx.x = class * tiles_per_class + tile, every
    // tile holds rows of one class and reduces over that class's taps only (3x3: 1, 2, 2, 4 of 9 taps; 1x1: one class, the
    // other three receive nothing).  Without this 3/4 of the rows of every 128-row tile were zero-filled.
    const bool par = MODE == DGRAD && d.stride == 2;
    int py = 0, px = 0, Hh = d.Hi, Wh = d.Wi, r0 = 0, s0 = 0, nr = d.kh, nsx = d.kw, tstep = 1, mtile = bx;
    if (par) {
        // a 1-tap filter axis has ONE non-empty parity (the epilogue zero-fills the sibling pixels); classes = npy * npx
        const int npy = d.kh >= 2 ? 2 : 1, npx = d.kw >= 2 ? 2 : 1;
        const int tpc = gx / (npy * npx), cls = bx / tpc;
        mtile = bx - cls * tpc;
        py = npy == 2 ? cls / npx : (d.pad & 1); px = npx == 2 ? cls % npx : (d.pad & 1); Hh = d.Hi >> 1; Wh = d.Wi >> 1;
        r0 = (py + d.pad) & 1; s0 = (px + d.pad) & 1;
        nr = (d.kh - r0 + 1) >> 1; nsx = (d.kw - s0 + 1) >> 1; tstep = 2;
    }
    const int Mrows = MODE == FWD ? d.B * d.Ho * d.Wo : (MODE == DGRAD ? d.B * Hh * Wh : d.Cout);
    const int ldo = MODE == FWD ? d.Cout : (MODE == DGRAD ? d.Cin : Kfull);
    const int Kred = MODE == FWD ? Kfull : (MODE == DGRAD ? nr * nsx * d.Cout : d.B * d.Ho * d.Wo);
    const int m0 = mtile * BM, n0 = blockIdx.y * BN;
    const int nkb_total = (Kred + BK - 1) / BK;
    if (par) kb_per_split = (nkb_total + (int)gridDim.z - 1) / (int)gridDim.z;      // the classes have different reduction lengths
    const int kb_begin = blockIdx.z * kb_per_split;
    const int nkb = max(0, min(kb_begin + kb_per_split, nkb_total) - kb_begin);
    // output row of tile row `row` (identity except for the parity classes)
    auto out_row = [&](int row) {
        if (!par) return row;
        const int b = row / (Hh * Wh), rem = row - b * (Hh * Wh);
        const int hh = rem / Wh, wh = rem - hh * Wh;
        return (b * d.Hi + 2 * hh + py) * d.Wi + 2 * wh + px;
    };
    // input pixels of the parities no tap reaches get zeros (non-accumulating calls): written by the thread that stores
    // the sibling pixel of the same 2x2 cell
    const bool fill_y = par && d.kh < 2 && !accumulate, fill_x = par && d.kw < 2 && !accumulate;
    auto zero_siblings = [&](int orow, int col) {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        const int dyr = (py ? -1 : 1) * d.Wi, dxr = px ? -1 : 1;
        if (fill_x) *reinterpret_cast<float4*>(O + (size_t)(orow + dxr) * ldo + col) = z;
        if (fill_y) *reinterpret_cast<float4*>(O + (size_t)(orow + dyr) * ldo + col) = z;
        if (fill_x && fill_y) *reinterpret_cast<float4*>(O + (size_t)(orow + dyr + dxr) * ldo + col) = z;
    };

    DBOA_TL(1);
    const int wg = warp >> 2;                              // warpgroup: tile rows 64 wg .. 64 wg + 63
    float acc[32], blk[32];                                // running total (round-to-nearest adds), accumulator of one k-block
#pragma unroll
    for (int q = 0; q < 32; ++q) { acc[q] = 0.f; blk[q] = 0.f; }

    {
        // =====================================================================================
        // loaders (8 warps): global -> registers (two k-blocks ahead) -> hi/lo split -> shared memory stage
        // FWD / DGRAD: the 128-row operand is pixel-major.  Warp w owns the 8-row groups 2w, 2w+1; lane = (row lr8, chunk
        // pair cpair): one LDG.128 of a warp covers 8 rows x 64 contiguous bytes (whole sectors), and the 8 lanes of one
        // shared-memory store phase fill the 8 rows of one core matrix (conflict free).  Register slot q*2 + h holds
        // row group 2w + q, 16-byte k-chunk h*4 + cpair.
        // =====================================================================================
        const int lr8 = lane & 7, cpair = lane >> 3;
        bool avalid[2] = {false, false};
        int ph[2] = {0, 0}, pw[2] = {0, 0};                // FWD: hi0, wi0 (top-left of the window); DGRAD: hi, wi
        int bq[2] = {0, 0};                                // sample of the row
        const float* pb[2] = {P, P};
        if (MODE != WGRAD) {
            const int HW = MODE == FWD ? d.Ho * d.Wo : Hh * Wh, Wd = MODE == FWD ? d.Wo : Wh;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int arow = m0 + (warp * 2 + q) * 8 + lr8;
                avalid[q] = arow < Mrows;
                if (avalid[q]) {
                    const int b = arow / HW, rem = arow - b * HW;
                    const int h = rem / Wd, w_ = rem - h * Wd;
                    bq[q] = b;
                    if (MODE == FWD) { ph[q] = h * d.stride - d.pad; pw[q] = w_ * d.stride - d.pad; pb[q] = P + (size_t)b * d.Hi * d.Wi * d.Cin; }
                    else { ph[q] = tstep * h + py; pw[q] = tstep * w_ + px; pb[q] = P + (size_t)b * d.Ho * d.Wo * d.Cout; }
                }
            }
        }
        // byte offset of (row group 2w + q, k-chunk h*4 + cpair, row lr8) in a stage tile: + q * GROUP_BYTES + h * 4 * CORE_BYTES
        const uint32_t a_off = (uint32_t)(warp * 2) * GROUP_BYTES + (uint32_t)cpair * CORE_BYTES + (uint32_t)lr8 * 16;
        // FWD: the weight tile is K-major too: row group w, chunks h*4 + cpair  ->  register slot h
        const uint32_t b_off = (uint32_t)warp * GROUP_BYTES + (uint32_t)cpair * CORE_BYTES + (uint32_t)lr8 * 16;
        // WGRAD: column tile -> (tap, ci0)
        const int wtap = MODE == WGRAD ? n0 / d.Cin : 0, wci0 = MODE == WGRAD ? n0 - wtap * d.Cin : 0;
        const int wr = wtap / d.kw, wsx = wtap - wr * d.kw;
        // reduction cursor of the two operand streams (tap row, tap column, channel offset): k-blocks are fetched in order,
        // so the im2col decode is an increment, not a division, per k-block
        const int Cred = MODE == DGRAD ? d.Cout : d.Cin;
        struct Cursor { int r, s, c; };
        // (r, s) count the taps of this CTA's tap set: filter tap = (r0 + tstep * r, s0 + tstep * s), nsx taps per filter row
        auto make_cursor = [&](int kb) { Cursor c; const int k0 = kb * BK, tap = k0 / Cred; c.c = k0 - tap * Cred; c.r = tap / max(nsx, 1); c.s = tap - c.r * max(nsx, 1); return c; };
        auto advance = [&](Cursor& c) { c.c += BK; if (c.c >= Cred) { c.c = 0; if (++c.s == nsx) { c.s = 0; ++c.r; } } };
        Cursor ca = make_cursor(kb_begin), cb = ca;
        int kb_a = kb_begin, kb_b = kb_begin;              // next k-block of each stream

        // XOP: the second source at the same element (residual / y_c), element offsets (-1: padding) and the channel base
        const float* xsrc = XF >= 2 && XF <= 3 ? e.res : e.y_c;
        auto fetch_a = [&](float4 (&ra)[4], float4 (&rx)[4], long long (&roff)[2], int& rch) {
            if (XOP) rch = ca.c;
            if (MODE == FWD) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int hi = ph[q] + ca.r, wi = pw[q] + ca.s;
                    const bool inb = avalid[q] && (unsigned)hi < (unsigned)d.Hi && (unsigned)wi < (unsigned)d.Wi;
                    const float* src = pb[q] + ((size_t)hi * d.Wi + wi) * d.Cin + ca.c + cpair * 4;
                    ra[q * 2] = inb ? ldg4(src) : make_float4(0.f, 0.f, 0.f, 0.f);
                    ra[q * 2 + 1] = inb ? ldg4(src + 16) : make_float4(0.f, 0.f, 0.f, 0.f);
                    if (XOP) roff[q] = inb ? (long long)(src - P) : -1;
                    if (XF >= 2 && XF <= 3 && inb) { rx[q * 2] = ldg4(xsrc + (src - P)); rx[q * 2 + 1] = ldg4(xsrc + (src - P) + 16); }
                }
            } else if (MODE == DGRAD) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int th = ph[q] + d.pad - (r0 + tstep * ca.r), tw = pw[q] + d.pad - (s0 + tstep * ca.s);
                    bool inb = avalid[q] && th >= 0 && tw >= 0;
                    int ho = th, wo = tw;
                    if (d.stride != 1) {
                        ho = th / d.stride; wo = tw / d.stride;
                        inb = inb && (ho * d.stride == th) && (wo * d.stride == tw);
                    }
                    inb = inb && ho < d.Ho && wo < d.Wo;
                    const float* src = pb[q] + ((size_t)ho * d.Wo + wo) * d.Cout + ca.c + cpair * 4;
                    ra[q * 2] = inb ? ldg4(src) : make_float4(0.f, 0.f, 0.f, 0.f);
                    ra[q * 2 + 1] = inb ? ldg4(src + 16) : make_float4(0.f, 0.f, 0.f, 0.f);
                    if (XOP) roff[q] = inb ? (long long)(src - P) : -1;
                    if (XDG && inb) { rx[q * 2] = ldg4(xsrc + (src - P)); rx[q * 2 + 1] = ldg4(xsrc + (src - P) + 16); }
                }
            } else {
                // A'[m=co][k=pix] = dY[pix][co]: rows of 128 consecutive co, one row per pixel (transposed by the store)
                const int k0 = kb_a * BK;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int idx = tid + NPROD * j, k = idx >> 5, cv = idx & 31;
                    const int pix = k0 + k, co = m0 + cv * 4;
                    ra[j] = (pix < Kred && co < d.Cout) ? ldg4(P + (size_t)pix * d.Cout + co) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
            ++kb_a;
            if (MODE != WGRAD) advance(ca);
        };
        auto fetch_b = [&](float4 (&rb)[2]) {
            const int k0 = kb_b * BK;
            if (MODE == FWD) {
                const float* wrow = Q + (size_t)(n0 + warp * 8 + lr8) * Kfull + k0 + cpair * 4;
                rb[0] = ldg4(wrow);
                rb[1] = ldg4(wrow + 16);
            } else if (MODE == DGRAD) {
                // B[n=ci][k=co] = W[co][tap][ci]: rows of 64 consecutive ci, one row per co (transposed by the store)
                // thread = (k = warp*4 + (lane & 3), nv = j*8 + (lane >> 3)*2 + ((lane >> 2) & 1)): bank-conflict-free transposing store
                const int tap = (r0 + tstep * cb.r) * d.kw + (s0 + tstep * cb.s);
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int k = warp * 4 + (lane & 3), nv = j * 8 + (lane >> 3) * 2 + ((lane >> 2) & 1);
                    rb[j] = ldg4(Q + (size_t)(cb.c + k) * Kfull + (size_t)tap * d.Cin + n0 + nv * 4);
                }
            } else {
                // B'[n=ci][k=pix] = X[pixel shifted by the tap][ci0 + n]
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int idx = tid + NPROD * j, k = idx >> 4, nv = idx & 15;
                    const int pix = k0 + k;
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (pix < Kred) {
                        const int b = pix / (d.Ho * d.Wo), rem = pix - b * d.Ho * d.Wo;
                        const int ho = rem / d.Wo, wo = rem - ho * d.Wo;
                        const int hi = ho * d.stride - d.pad + wr, wi = wo * d.stride - d.pad + wsx;
                        if ((unsigned)hi < (unsigned)d.Hi && (unsigned)wi < (unsigned)d.Wi)
                            v = ldg4(Q + (((size_t)b * d.Hi + hi) * d.Wi + wi) * d.Cin + wci0 + nv * 4);
                    }
                    rb[j] = v;
                }
            }
            ++kb_b;
            if (MODE == DGRAD) advance(cb);
        };
        // XFWD: relu(gn(x) [+ res | + gn2(res)]), materialised into a_out by the CTAs of the first column tile; XDG: GroupNorm
        // backward dy = rstd (dz gamma - m1 - x^ m2), x^ = (y_c - mean) rstd, materialised into dy_out the same way.  Padding stays 0.
        const int Cop = MODE == FWD ? d.Cin : d.Cout, gsz = Cop / 4;
        float* mat = XFWD ? e.a_out : e.dy_out;
        auto xform = [&](float4 v, float4 r, int q, int ch) {
            const int gi = bq[q] * 4 + ch / gsz;
            const float2 t0 = s_gn[0][gi];
            float a[4] = {v.x, v.y, v.z, v.w}, x2[4] = {r.x, r.y, r.z, r.w};
            if (XFWD) {
                const float4 g4 = ldg4(e.gamma + ch), b4 = ldg4(e.beta + ch);
                const float gg[4] = {g4.x, g4.y, g4.z, g4.w}, bb[4] = {b4.x, b4.y, b4.z, b4.w};
                float g2[4] = {0.f, 0.f, 0.f, 0.f}, b2[4] = {0.f, 0.f, 0.f, 0.f};
                float2 t1 = make_float2(0.f, 0.f);
                if (XF == 3) {
                    const float4 h4 = ldg4(e.gamma2 + ch), c4 = ldg4(e.beta2 + ch);
                    g2[0] = h4.x; g2[1] = h4.y; g2[2] = h4.z; g2[3] = h4.w; b2[0] = c4.x; b2[1] = c4.y; b2[2] = c4.z; b2[3] = c4.w;
                    t1 = s_gn[1][gi];
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float t = (a[i] - t0.x) * t0.y * gg[i] + bb[i];
                    if (XF == 2) t += x2[i];
                    if (XF == 3) t += (x2[i] - t1.x) * t1.y * g2[i] + b2[i];
                    a[i] = fmaxf(t, 0.f);
                }
            } else {
                const float4 g4 = ldg4(e.gamma_c + ch);
                const float gg[4] = {g4.x, g4.y, g4.z, g4.w};
                const float2 m = s_gn[1][gi];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float xh = (x2[i] - t0.x) * t0.y;
                    a[i] = t0.y * (a[i] * gg[i] - m.x - xh * m.y);
                }
            }
            return make_float4(a[0], a[1], a[2], a[3]);
        };
        auto stash = [&](int s, float4 (&ra)[4], const float4 (&rb)[2], const float4 (&rx)[4], const long long (&roff)[2], int rch) {
            if (XOP) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int q = j >> 1, ch = rch + cpair * 4 + (j & 1) * 16;
                    if (roff[q] >= 0) {
                        ra[j] = xform(ra[j], rx[j], q, ch);
                        if (mat != nullptr && blockIdx.y == 0) *reinterpret_cast<float4*>(mat + roff[q] + (j & 1) * 16) = ra[j];
                    }
                }
            }
            if (MODE != WGRAD) {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    split_store4(sm.a_hi[s], sm.a_lo[s], a_off + (j >> 1) * GROUP_BYTES + (j & 1) * 4 * CORE_BYTES, ra[j]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int idx = tid + NPROD * j;
                    split_store_t(sm.a_hi[s], sm.a_lo[s], (idx & 31) * 4, idx >> 5, ra[j]);
                }
            }
            if (MODE == FWD) {
                split_store4(sm.b_hi[s], sm.b_lo[s], b_off, rb[0]);
                split_store4(sm.b_hi[s], sm.b_lo[s], b_off + 4 * CORE_BYTES, rb[1]);
            } else if (MODE == DGRAD) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int k = warp * 4 + (lane & 3), nv = j * 8 + (lane >> 3) * 2 + ((lane >> 2) & 1);
                    split_store_t_rot(sm.b_hi[s], sm.b_lo[s], nv * 4, k, rb[j], lane >> 3);
                }
            } else {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int idx = tid + NPROD * j;
                    split_store_t(sm.b_hi[s], sm.b_lo[s], (idx & 15) * 4, idx >> 4, rb[j]);
                }
            }
        };

        // Programmatic dependent launch: everything above (index set-up) and -- for the forward and data-gradient products --
        // the first WEIGHT tiles do not depend on the previous kernel in the stream and overlap its tail; activations are
        // touched only after the wait.  (Weights are never written by the kernel that immediately precedes a convolution:
        // optimizer updates are followed by a normally serialized launch.)
        float4 ra[STAGES][4], rb[STAGES][2], rx[STAGES][4];
        long long roff[STAGES][2];
        int rch[STAGES];
        if (MODE != WGRAD) {
#pragma unroll
            for (int f = 0; f < STAGES; ++f)
                if (f < nkb) fetch_b(rb[f]);
        }
        DBOA_TL(2);
        pdl_wait();
        pdl_trigger();
        DBOA_TL(3);
        if (XOP) {
            // per (sample, group) tables of the transform, from the producers' fixed-point sums
            const double n = (double)d.Ho * d.Wo * Cop / 4;        // XFWD: elements of one group of the operand (its producer's output)
            const double nx = (double)d.Hi * d.Wi * d.Cin / 4;
            for (int i = tid; i < d.B * 4; i += NT) {
                if (XFWD) {
                    for (int k = 0; k < (XF == 3 ? 2 : 1); ++k) {
                        const long long* a = k ? e.acc2_in : e.acc_in;
                        const double mean = (double)a[i * 2] / FIX_FWD / nx, var = fmax((double)a[i * 2 + 1] / FIX_FWD / nx - mean * mean, 0.0);
                        const float rstd = (float)(1.0 / sqrt(var + 1e-5));
                        s_gn[k][i] = make_float2((float)mean, rstd);
                        float* so = k ? e.stats2_out : e.stats_out;
                        if (so != nullptr && (blockIdx.x | blockIdx.y | blockIdx.z) == 0) { so[i * 2] = (float)mean; so[i * 2 + 1] = rstd; }
                    }
                } else {
                    s_gn[0][i] = make_float2(e.stats_c[i * 2], e.stats_c[i * 2 + 1]);
                    s_gn[1][i] = make_float2((float)((double)e.sums_c[i * 2] / FIX_BWD / n), (float)((double)e.sums_c[i * 2 + 1] / FIX_BWD / n));
                }
            }
            __syncthreads();
        }
#pragma unroll
        for (int f = 0; f < STAGES; ++f)
            if (f < nkb) { fetch_a(ra[f], rx[f], roff[f], rch[f]); if (MODE == WGRAD) fetch_b(rb[f]); }
        // Per k-block: stash stage s, barrier, issue the MMAs of stage s, issue the loads of k-block it + 2, wait for the MMAs and
        // add them to the total.  Stage s was last read by the MMAs of k-block it - 2, which both warpgroups waited for before
        // the previous barrier.
        const uint64_t a_step = (uint64_t)((wg * 8 * GROUP_BYTES) >> 4);
        for (int it0 = 0; it0 < nkb; it0 += STAGES) {
#pragma unroll
            for (int f = 0; f < STAGES; ++f) {
                const int it = it0 + f;
                if (it < nkb) {
                    const int s = f;                                                              // stage == register set
                    DBOA_TLC(it, 0);
                    stash(s, ra[f], rb[f], rx[f], roff[f], rch[f]);
                    DBOA_TLC(it, 2);
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> async-proxy (wgmma) reads
                    __syncthreads();
                    DBOA_TLC(it, 3);
                    if (it == 0) DBOA_TL(4);
                    const uint64_t dah = make_desc(smem_u32(sm.a_hi[s])) + a_step, dal = make_desc(smem_u32(sm.a_lo[s])) + a_step;
                    const uint64_t dbh = make_desc(smem_u32(sm.b_hi[s])), dbl = make_desc(smem_u32(sm.b_lo[s]));
                    constexpr uint64_t KSTEP = (2 * CORE_BYTES) >> 4;      // 8 tf32 = two 16-byte chunks along K, in descriptor units
                    fence_operand(blk);
                    wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < BK / 8; ++kk) {
                        wgmma_tf32(blk, dah + kk * KSTEP, dbh + kk * KSTEP, kk > 0);
                        wgmma_tf32(blk, dah + kk * KSTEP, dbl + kk * KSTEP, 1);
                        wgmma_tf32(blk, dal + kk * KSTEP, dbh + kk * KSTEP, 1);
                    }
                    wgmma_commit();
                    if (it + STAGES < nkb) { fetch_a(ra[f], rx[f], roff[f], rch[f]); fetch_b(rb[f]); }                    // in flight behind the MMAs
                    // the k-block's MMAs complete inside this straight-line block: an accumulator that stays in flight across the
                    // unrolled loop's branches gets register copies inside the asynchronous region, and ptxas then serialises
                    // every wgmma (C7515)
                    wgmma_wait_all();
                    fence_operand(blk);
#pragma unroll
                    for (int q = 0; q < 32; ++q) acc[q] += blk[q];
                    DBOA_TLC(it, 4);
                }
            }
        }
    }
    DBOA_TL(5);
    __syncthreads();                                       // every MMA of this CTA has completed: the A tiles are free
    DBOA_TL(6);

    // ---- epilogue: accumulator fragments -> shared memory (row-major tile) -> row-contiguous global stores
    const int nz = gridDim.z;
    float* red = reinterpret_cast<float*>(sm.a_hi[0]);    // 128 rows x RED_LD floats (34 KB) over the A tiles
    {
        const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2), col = (lane & 3) * 2;
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const int r = row + 8 * ((i >> 1) & 1), c = col + 8 * (i >> 2);
            *reinterpret_cast<float2*>(red + r * RED_LD + c) = make_float2(acc[i], acc[i + 1]);
        }
    }
    DBOA_TL(7);
    // Fused epilogues.  A thread's columns are fixed (v & 15 does not change as v advances by NT) and its rows ascend, so the sums
    // are kept per thread and flushed as fixed-point atomics (exact integer addition: order independent) when the sample changes.
    constexpr bool FSTAT = XF >= 0 && XF <= 3;
    const bool prep = XDG && e.mask != nullptr;
    const int HWo = MODE == FWD ? d.Ho * d.Wo : d.Hi * d.Wi, gs_out = (MODE == FWD ? d.Cout : d.Cin) / 4;
    int cur_b = -1;
    double st0[2] = {0.0, 0.0}, st1[2] = {0.0, 0.0}, dg[2][4] = {}, db[2][4] = {};
    int col_t = -1;
    auto flush_b = [&]() {
        if (cur_b < 0) return;
        const int gi = (cur_b * 4 + col_t / gs_out) * 2;
        if (FSTAT) { add_fixed(e.acc_out + gi, st0[0], FIX_FWD); add_fixed(e.acc_out + gi + 1, st1[0], FIX_FWD); }
        if (XDG) for (int j = 0; j < 2; ++j) if (prep && j < e.nprep) { add_fixed(e.prep_sums[j] + gi, st0[j], FIX_BWD); add_fixed(e.prep_sums[j] + gi + 1, st1[j], FIX_BWD); }
        st0[0] = st0[1] = st1[0] = st1[1] = 0.0;
    };
    auto post = [&](int orow, int col, float4 q) {
        if (!FSTAT && !XDG) return q;
        if (XDG) {
            if (e.addend != nullptr) { const float4 a = *reinterpret_cast<const float4*>(e.addend + (size_t)orow * ldo + col); q.x += a.x; q.y += a.y; q.z += a.z; q.w += a.w; }
            if (!prep) return q;
            const float4 m = *reinterpret_cast<const float4*>(e.mask + (size_t)orow * ldo + col);
            q.x = m.x > 0.f ? q.x : 0.f; q.y = m.y > 0.f ? q.y : 0.f; q.z = m.z > 0.f ? q.z : 0.f; q.w = m.w > 0.f ? q.w : 0.f;
        }
        const int b = orow / HWo;
        if (b != cur_b) { flush_b(); cur_b = b; }
        col_t = col;
        const float v[4] = {q.x, q.y, q.z, q.w};
        if (FSTAT) {
#pragma unroll
            for (int i = 0; i < 4; ++i) { st0[0] += v[i]; st1[0] += (double)v[i] * v[i]; }
        } else {
            for (int j = 0; j < 2; ++j) {
                if (j >= e.nprep) break;
                const float4 y4 = *reinterpret_cast<const float4*>(e.prep_y[j] + (size_t)orow * ldo + col);
                const float4 g4 = ldg4(e.prep_gamma[j] + col);
                const float2 ms = *reinterpret_cast<const float2*>(e.prep_stats[j] + (size_t)(b * 4 + col / gs_out) * 2);
                const float yy[4] = {y4.x, y4.y, y4.z, y4.w}, gg[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const double xh = ((double)yy[i] - ms.x) * ms.y;
                    st0[j] += (double)v[i] * gg[i]; st1[j] += (double)v[i] * gg[i] * xh;
                    dg[j][i] += v[i] * xh; db[j][i] += v[i];
                }
            }
        }
        return q;
    };
    auto flush_all = [&]() {
        flush_b();
        if (prep && col_t >= 0)
            for (int j = 0; j < e.nprep && j < 2; ++j)
#pragma unroll
                for (int i = 0; i < 4; ++i) { add_fixed(e.prep_dgb[j] + (size_t)(col_t + i) * 2, dg[j][i], FIX_BWD); add_fixed(e.prep_dgb[j] + (size_t)(col_t + i) * 2 + 1, db[j][i], FIX_BWD); }
    };
    if (nz == 1) {
        __syncthreads();
        for (int v = tid; v < BM * (BN / 4); v += NT) {               // 16 lanes write one 256-byte output row
            const int lr = v >> 4, c4 = (v & 15) * 4;
            const int row = m0 + lr;
            if (row < Mrows) {
                float4 q = *reinterpret_cast<const float4*>(red + lr * RED_LD + c4);
                const int orow = out_row(row);
                float4* dst = reinterpret_cast<float4*>(O + (size_t)orow * ldo + n0 + c4);
                if (accumulate) { const float4 c = *dst; q.x += c.x; q.y += c.y; q.z += c.z; q.w += c.w; }
                q = post(orow, n0 + c4, q);
                *dst = q;
                if (fill_x || fill_y) zero_siblings(orow, n0 + c4);
            }
        }
    } else {
        cg::cluster_group cluster = cg::this_cluster();
        cluster.sync();
        DBOA_TL(8);
        const int rank = (int)cluster.block_rank();
        const int rows_per = BM / nz;                                 // nz is a power of two <= 16
        for (int v = tid; v < rows_per * (BN / 4); v += NT) {
            const int lr = rank * rows_per + (v >> 4), c4 = (v & 15) * 4;
            const int row = m0 + lr;
            if (row >= Mrows) continue;
            const int orow = out_row(row);
            float4* dst = reinterpret_cast<float4*>(O + (size_t)orow * ldo + n0 + c4);
            if (fill_x || fill_y) zero_siblings(orow, n0 + c4);
            float4 sacc = accumulate ? *dst : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int zb = 0; zb < 16; zb += 8) {                      // 8 remote loads in flight, then added in the order z = 0..nz-1
                if (zb < nz) {
                    float4 q[8];
#pragma unroll
                    for (int z = 0; z < 8; ++z)
                        if (zb + z < nz) q[z] = *reinterpret_cast<const float4*>(cluster.map_shared_rank(red, zb + z) + lr * RED_LD + c4);
#pragma unroll
                    for (int z = 0; z < 8; ++z)
                        if (zb + z < nz) { sacc.x += q[z].x; sacc.y += q[z].y; sacc.z += q[z].z; sacc.w += q[z].w; }
                }
            }
            *dst = post(orow, n0 + c4, sacc);
        }
        DBOA_TL(9);
        cluster.sync();                                               // peers may still be reading this CTA's tile
    }
    if (FSTAT || prep) flush_all();
    DBOA_TL(10);
}

template <int MODE, int XF = -1>
static int launch(const float* p, const float* q, float* o, const ConvDims& d, int rows, int cols, int kred, int accumulate, cudaStream_t st,
                  bool pdl, const Ext& e = Ext()) {
    int mtiles = ceil_div(rows, BM);
    if (MODE == DGRAD && d.stride == 2) {                // parity classes of B*Hi/2*Wi/2 rows, longest tap set decides the split
        const int ncls = (d.kh >= 2 ? 2 : 1) * (d.kw >= 2 ? 2 : 1);
        mtiles = ncls * ceil_div(d.B * (d.Hi / 2) * (d.Wi / 2), BM);
        kred = ((d.kh + 1) / 2) * ((d.kw + 1) / 2) * d.Cout;
    }
    mtiles *= d.groups;                                  // every group's tiles count towards the split-K sizing
    const int nkb = (kred + BK - 1) / BK;
    const int tiles = mtiles * (cols / BN);
    // K-slices per tile (cluster size): a power of two <= 8 (the portable cluster size) that keeps the grid within about one wave; a split must
    // leave at least `min_kb` k-blocks per CTA, since the cluster barrier and DSMEM reduction of a split tile cost several k-blocks.
    static const int min_kb = [] { const char* e = getenv("DBOA_TC_MINKB"); int v = e ? atoi(e) : 2; return v < 1 ? 1 : v; }();
    int ns = 1;
    const int slots = num_sms();                          // one resident CTA per SM (~150-215 registers x 256 threads)
    while (ns < 8 && tiles * ns * 2 <= slots + tiles && nkb / (ns * 2) >= min_kb) ns *= 2;
    const int per = (nkb + ns - 1) / ns;
    const size_t smem = sizeof(Smem) + 128;
    auto kernel = conv_tf32x3_kernel<MODE, XF>;
    if constexpr (XF < 0)                                 // the fused variants serve one group only
        if (d.groups > 1) kernel = conv_tf32x3_kernel<MODE, XF, true>;
    return launch_ex(kernel, dim3(mtiles, cols / BN, ns), dim3(NT), smem, st, dim3(1, 1, ns), pdl, p, q, o, d, per, accumulate, e);
}

static bool shape_ok(const ConvDims& d) {
    return d.groups >= 1 && d.Cin % 64 == 0 && d.Cout % 64 == 0 && d.Kpitch == d.kh * d.kw * d.Cin;
}

}  // namespace tc

#ifdef DBOA_TIMELINE
extern "C" int dboa_debug_set_timeline(unsigned long long* buf) {
    return cudaMemcpyToSymbol(tc::g_timeline, &buf, sizeof(buf)) == cudaSuccess ? 0 : -3;
}
#endif

int conv_tc_fwd(const float* x, const float* w, float* y, const ConvDims& d, cudaStream_t st, bool pdl) {
    if (g_tc_mode == 0 || !tc::shape_ok(d)) return DBOA_ERR_UNSUPPORTED;
    return tc::launch<tc::FWD>(x, w, y, d, d.B * d.Ho * d.Wo, d.Cout, d.kh * d.kw * d.Cin, 0, st, pdl);
}
int conv_tc_dgrad(const float* dy, const float* w, float* dx, const ConvDims& d, int accumulate, cudaStream_t st, bool pdl) {
    if (g_tc_mode < 2 || !tc::shape_ok(d)) return DBOA_ERR_UNSUPPORTED;
    if (d.stride == 2 && ((d.Hi | d.Wi) & 1)) return DBOA_ERR_UNSUPPORTED;       // the parity-class enumeration needs even extents
    return tc::launch<tc::DGRAD>(dy, w, dx, d, d.B * d.Hi * d.Wi, d.Cin, d.kh * d.kw * d.Cout, accumulate, st, pdl);
}
int conv_tc_wgrad(const float* dy, const float* x, float* dw, const ConvDims& d, cudaStream_t st, bool pdl) {
    if (g_tc_mode < 2 || !tc::shape_ok(d)) return DBOA_ERR_UNSUPPORTED;
    return tc::launch<tc::WGRAD>(dy, x, dw, d, d.Cout, d.kh * d.kw * d.Cin, d.B * d.Ho * d.Wo, 1, st, pdl);
}

// weight gradient on the tensor cores whatever the plan's mode (C ABI dboa_conv2d_wgrad_tma); dw is accumulated
int conv_wgrad_tc(const float* dy, const float* x, float* dw, const ConvDims& d, cudaStream_t st) {
    if (!tc::shape_ok(d)) return DBOA_ERR_UNSUPPORTED;
    return tc::launch<tc::WGRAD>(dy, x, dw, d, d.Cout, d.kh * d.kw * d.Cin, d.B * d.Ho * d.Wo, 1, st, false);
}

bool conv_fused_ok(const FusedConv& f) {
    return f.Cin % 64 == 0 && f.Cout % 64 == 0 && (f.k == 1 || f.k == 3) && (f.stride == 1 || f.stride == 2) && f.mode >= 0 && f.mode <= 3;
}
static bool fused_batch_ok(int B) { return B >= 1 && B <= 64; }      // the per-(sample, group) table in shared memory holds 64 samples

// one launch per problem: y = conv(T(x), w), T of FusedConv::mode applied by the loader, statistics of y from the epilogue
int conv_fused_fwd(const FusedConv* fc, int nprob, int B, cudaStream_t st, bool pdl) {
    if (!fused_batch_ok(B)) return DBOA_ERR_UNSUPPORTED;
    for (int i = 0; i < nprob; ++i) {
        const FusedConv& f = fc[i];
        if (!conv_fused_ok(f)) return DBOA_ERR_UNSUPPORTED;
        ConvDims d;
        d.B = B; d.Hi = d.Wi = f.Hi; d.Cin = f.Cin; d.Cout = f.Cout; d.kh = d.kw = f.k; d.stride = f.stride; d.pad = f.pad;
        d.Ho = d.Wo = (f.Hi + 2 * f.pad - f.k) / f.stride + 1; d.Kpitch = f.k * f.k * f.Cin;
        tc::Ext e = {};
        e.res = f.res; e.acc_in = reinterpret_cast<const long long*>(f.part_in); e.acc2_in = reinterpret_cast<const long long*>(f.part2_in);
        e.gamma = f.gamma; e.beta = f.beta; e.gamma2 = f.gamma2; e.beta2 = f.beta2;
        e.a_out = f.a_out; e.stats_out = f.stats_out; e.stats2_out = f.stats2_out; e.acc_out = reinterpret_cast<long long*>(f.part_out);
        const int rows = B * d.Ho * d.Wo, K = d.Kpitch;
        int r;
        switch (f.mode) {
            case 0: r = tc::launch<tc::FWD, 0>(f.x, f.w, f.y, d, rows, d.Cout, K, 0, st, pdl, e); break;
            case 1: r = tc::launch<tc::FWD, 1>(f.x, f.w, f.y, d, rows, d.Cout, K, 0, st, pdl, e); break;
            case 2: r = tc::launch<tc::FWD, 2>(f.x, f.w, f.y, d, rows, d.Cout, K, 0, st, pdl, e); break;
            default: r = tc::launch<tc::FWD, 3>(f.x, f.w, f.y, d, rows, d.Cout, K, 0, st, pdl, e); break;
        }
        if (r != DBOA_OK) return r;
    }
    return DBOA_OK;
}

bool dgrad_fused_ok(const ConvDims& d) {
    return tc::shape_ok(d) && d.stride == 1 && (d.kh == 1 || d.kh == 3) && d.kh == d.kw && d.pad == d.kh / 2 && d.Hi == d.Ho && d.B <= 64;
}

// data gradient with GroupNorm_c backward on load and the addend / ReLU mask / next GroupNorm-backward sums in the epilogue
int dgrad_fused(const DgradFused& f, const ConvDims& d, cudaStream_t st, bool pdl) {
    if (!dgrad_fused_ok(d) || f.nprep < 0 || f.nprep > 2) return DBOA_ERR_UNSUPPORTED;
    tc::Ext e = {};
    e.y_c = f.y_c; e.stats_c = f.stats_c; e.sums_c = reinterpret_cast<const long long*>(f.sums_c); e.gamma_c = f.gamma_c; e.dy_out = f.dy_out;
    e.addend = f.addend; e.mask = f.mask; e.nprep = f.mask ? f.nprep : 0;
    for (int j = 0; j < 2; ++j) {
        e.prep_y[j] = f.prep[j].y; e.prep_stats[j] = f.prep[j].stats; e.prep_gamma[j] = f.prep[j].gamma;
        e.prep_sums[j] = reinterpret_cast<long long*>(f.prep[j].sums); e.prep_dgb[j] = reinterpret_cast<long long*>(f.prep[j].dgb);
    }
    return tc::launch<tc::DGRAD, tc::XD>(f.dz, f.w, f.out, d, d.B * d.Hi * d.Wi, d.Cin, d.kh * d.kw * d.Cout, f.mask ? 0 : f.accumulate, st, pdl, e);
}

int conv1x1_tc_fwd(const float* x, const float* w, float* y, int M, int Cin, int Cout, cudaStream_t st, bool pdl) {
    ConvDims d;
    d.B = 1; d.Hi = M; d.Wi = 1; d.Cin = Cin; d.Ho = M; d.Wo = 1; d.Cout = Cout; d.kh = 1; d.kw = 1; d.stride = 1; d.pad = 0; d.Kpitch = Cin;
    return conv_tc_fwd(x, w, y, d, st, pdl);
}

}  // namespace dboa
