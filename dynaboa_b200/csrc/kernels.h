// Internal launcher prototypes shared between the kernel translation units, the per-op C-ABI
// wrappers (cabi.cu) and the whole-network plan (hmr_plan.cu).  Not part of the public ABI.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include "../../include/dynaboa_b200.h"

namespace dboa {

// Grouped convolutions (several independent videos in one launch): `groups` blocks of B samples each, stored one after the
// other in the activations; group g uses the weights w + g * wstride (the weight gradient writes dw + g * wstride).
// `active`: bit g set means group g takes part; the CTAs of an idle group return before touching memory (grouped calls only).
struct ConvDims {
    int B, Hi, Wi, Cin, Ho, Wo, Cout, kh, kw, stride, pad, Kpitch;
    int groups = 1;
    long long wstride = 0;
    unsigned long long active = ~0ULL;
};

// ---- conv.cu (fp32 CUDA-core implicit GEMM)
int conv_fwd(const float* x, const float* w, float* y, const ConvDims& d, float* ws, size_t ws_floats, cudaStream_t st);
int conv_dgrad(const float* dy, const float* w, float* dx, const ConvDims& d, int accumulate, float* ws, size_t ws_floats, cudaStream_t st);
int conv_wgrad(const float* dy, const float* x, float* dw, const ConvDims& d, float* ws, size_t ws_floats, cudaStream_t st);

// ---- conv_tc.cu (wgmma TF32x3 implicit GEMM); returns DBOA_ERR_UNSUPPORTED when the shape is not taken
// `pdl`: launch with programmatic stream serialization.  The forward / data-gradient kernels prefetch WEIGHT tiles before
// their dependency wait, which is only safe when the preceding kernel in the stream does not write the weights (true inside
// the network plan; the stand-alone C-ABI wrappers pass false).
int conv_tc_fwd(const float* x, const float* w, float* y, const ConvDims& d, cudaStream_t st, bool pdl = true);
int conv_tc_dgrad(const float* dy, const float* w, float* dx, const ConvDims& d, int accumulate, cudaStream_t st, bool pdl = true);
int conv_tc_wgrad(const float* dy, const float* x, float* dw, const ConvDims& d, cudaStream_t st, bool pdl = true);
bool conv_tc_bwd_enabled();
bool conv_tc_wgrad_enabled();
int conv1x1_tc_fwd(const float* x, const float* w, float* y, int M, int Cin, int Cout, cudaStream_t st, bool pdl = true);
bool conv_tc_enabled();
void conv_tc_set_mode(int mode);                      // 0 off, 1 forward, 2 forward + dgrad + wgrad, 3 forward + dgrad

int conv_wgrad_tc(const float* dy, const float* x, float* dw, const ConvDims& d, cudaStream_t st);   // any mode; dw +=

// ---- fused convolutions (conv_tc.cu, same kernel with an operand transform on load and sums in the epilogue)
struct FusedConv {
    const float *x, *res, *w;                 // operand source (see `mode`), second source (modes 2, 3), weights [Cout][k*k*Cin]
    float *a_out, *stats_out, *stats2_out;    // optional tape stores: transformed operand, (mean, rstd) [B][4][2] of the operand's GroupNorm(s)
    const float *part_in, *part2_in;          // fixed-point (sum, sum of squares) long long [B][4][2] of x / res left by their producers
    const float *gamma, *beta, *gamma2, *beta2;
    float *y, *part_out;                      // raw output [B][Ho][Ho][Cout] and its statistics accumulators (ZEROED by the caller)
    int mode;                                 // 0: x as is; 1: relu(gn(x)); 2: relu(gn(x) + res); 3: relu(gn(x) + gn2(res))
    int Hi, Cin, Cout, k, stride, pad, Ho;    // square images
};
bool conv_fused_ok(const FusedConv& f);
int conv_fused_fwd(const FusedConv* f, int nprob, int B, cudaStream_t st, bool pdl);
int gn_acc_res_avgpool(const float* y, const float* res, const float* acc, const float* gamma, const float* beta, float* a_out, float* stats_out,
                       float* out, int B, int HW, int C, int ld, int ncopy, size_t copy_stride, cudaStream_t st);
// fused data gradient: GroupNorm backward of the operand on load, ReLU mask + the next GroupNorm backward's sums in the epilogue.
// All sums are 64-bit fixed point (long long, scale 2^28), zeroed by the caller.
struct DgradPrep {
    const float* y;            // raw output of the layer whose GroupNorm backward is prepared [B][H][W][C]
    const float* stats;        // its (mean, rstd) [B][4][2]
    const float* gamma;
    float* sums;               // long long [B][4][2]: sum q, sum q x^   (q = dz gamma)
    float* dgb;                // long long [C][2]: d gamma, d beta
};
struct DgradFused {
    const float *dz, *y_c, *w;                     // masked gradient w.r.t. GroupNorm_c's output, raw output of conv c, weights of conv c
    const float *stats_c, *sums_c, *gamma_c;       // GroupNorm_c: (mean, rstd), backward sums (long long), gamma
    float* dy_out;                                 // dy_c materialised for the weight gradient, or NULL
    const float* addend;                           // added to dX before the mask (shortcut gradient), or NULL
    float* out;                                    // mask == NULL: dX (accumulate: +=); else dz of the producing layer
    const float* mask;                             // post-activation output of the producing layer, or NULL
    DgradPrep prep[2];
    int nprep, accumulate;
};
bool dgrad_fused_ok(const ConvDims& d);
int dgrad_fused(const DgradFused& f, const ConvDims& d, cudaStream_t st, bool pdl);
int gn_bwd_prep(const float* dA, const float* mask, float* out, const DgradPrep& p, int B, int HW, int C, cudaStream_t st);
struct GnFinishItem;
int gn_dgb_finish(const GnFinishItem* items_dev, int n_items, const float* dgb, float* G, cudaStream_t st);

// ---- stem_wgrad.cu: 7x7 / stride-2 stem weight gradient: row-per-CTA partials + fixed-order reduction (stem_wgrad.cu); needs 64 * 147 floats of
// workspace per partial (DBOA_ERR_UNSUPPORTED for any other shape or without workspace)
bool stem_wgrad_ok(const ConvDims& d);
int stem_wgrad(const float* dy, const float* x, float* dw, const ConvDims& d, float* ws, size_t ws_floats, cudaStream_t st);

// ---- groupnorm.cu (single-launch cluster kernels)
size_t gn_partial_floats(int B, int HW, int C);     // forward scratch (none; kept for the C ABI)
size_t gn_bwd_partial_floats(int B, int HW, int C); // backward scratch: per-sample dgamma / dbeta rows
// out = relu?( gn(y) [+ res] ); writes (mean, rstd) to stats[B][4][2]
// backward: dz = dout * (mask_src > 0 if mask_src else 1); dy = GN backward; dgamma/dbeta accumulate (+=)
// Grouped (B = groups * bper samples): sample s uses gamma / beta + (s / bper) * pstride.  bper = B: one set for all.
int gn_fwd_fused(const float* y, const float* gamma, const float* beta, const float* res, float* out, float* stats, float* partial,
                 int B, int HW, int C, int relu, cudaStream_t st, int bper = 0, long long pstride = 0);
// defer = 1 (B > 1 only): leave the per-sample dgamma / dbeta rows in `partial` for gn_param_finish instead of reducing them here
// (required when bper < B: the rows of each group then go to that group's gradient through gn_param_finish)
int gn_bwd_fused(const float* dout, const float* mask_src, const float* y, const float* stats, const float* gamma, float* dy,
                 float* dgamma, float* dbeta, float* partial, int B, int HW, int C, cudaStream_t st, int defer = 0, int bper = 0,
                 long long pstride = 0);
int gn_prepare();                                   // the backward's cluster sync words (allocated once, before any capture)
struct GnFinishItem { long long g_off, b_off, cum_channels; int C; };
// rows of samples [g * B / groups, (g + 1) * B / groups) are added to G + g * pstride (groups whose `active` bit is set)
int gn_param_finish(const GnFinishItem* items_dev, int n_items, const float* rows, float* G, int B, cudaStream_t st, int groups = 1,
                    long long pstride = 0, unsigned long long active = ~0ULL);
// ---- norm_pool.cu
int relu_mask(const float* dout, const float* mask_src, float* dz, size_t n, cudaStream_t st);
int nchw_to_nhwc(const float* x, float* y, int B, int C, int H, int W, cudaStream_t st);
int maxpool3x3s2_fwd(const float* x, float* y, unsigned char* idx, int B, int H, int W, int C, cudaStream_t st);
int maxpool3x3s2_bwd(const float* dy, const unsigned char* idx, float* dx, int B, int H, int W, int C, cudaStream_t st);
// mean over HW -> out rows with leading dimension ld, replicated `ncopy` times `copy_stride` floats apart
int avgpool_fwd(const float* x, float* out, int B, int HW, int C, int ld, int ncopy, size_t copy_stride, cudaStream_t st);
int avgpool_bwd(const float* dxf, int ld, float* dx, int B, int HW, int C, cudaStream_t st);

// ---- head.cu
// Grouped variants: B = groups * (B / groups) rows, row b uses W / bias + (b / (B / groups)) * wstride.  Only the groups whose
// `active` bit is set are computed; the rows of the others are left as they were (linear_dgrad: unspecified).
// y[b][n] = (addend ? addend[b][n] : 0) + bias[n] + sum_k x[b][k] W[n][k];  pre <- y (before mask), post <- y*mask
int linear_fwd(const float* x, int ldx, const float* W, int ldw, const float* bias, const float* addend, int ld_add,
               const float* mask, float* pre, float* post, int ld_out, float* post2, int ld_out2,
               int B, int N, int K, cudaStream_t st, int groups = 1, long long wstride = 0, unsigned long long active = ~0ULL);
// dx[b][k] = sum_n dy[b][n] W[n][k] (k < K)
int linear_dgrad(const float* dy, int ldy, const float* W, int ldw, float* dx, int ldx, int B, int N, int K,
                 float* ws, size_t ws_floats, cudaStream_t st, int groups = 1, long long wstride = 0, unsigned long long active = ~0ULL);
// dW[n][k] += sum_r dy[r][n] x[r][k];  db[n] += sum_r dy[r][n].  The R rows are `R / B` slabs of B rows; group g reduces the
// rows g * B / groups .. (g + 1) * B / groups - 1 of every slab into dW / db + g * wstride (groups = 1: B is ignored)
int linear_wgrad(const float* dy, int ldy, const float* x, int ldx, float* dW, int ldw, float* db, int R, int N, int K, cudaStream_t st,
                 int groups = 1, int B = 0, long long wstride = 0, unsigned long long active = ~0ULL);
int rot6d_fwd_launch(const float* pose6d, float* rotmat, int n, cudaStream_t st);
int rot6d_bwd_launch(const float* pose6d, const float* drot, float* dpose, int n, cudaStream_t st);
int ew_mul(const float* a, const float* b, float* out, size_t n, cudaStream_t st);
int ew_add_rows(float* dst, int ld_dst, const float* a, int lda, const float* b, int ldb, int B, int n, cudaStream_t st);

// ---- dataprocess.cu (crop + anti-aliased resize + normalise, keypoint transform)
int crop_resize_normalize(const void* img, int is_u8, int H, int W, int ul_x, int ul_y, int Hc, const float* wx, const int* sx, int Tx,
                          const float* wy, const int* sy, int Ty, int res, const float mean[3], const float stdv[3], float* tmp, float* out,
                          cudaStream_t st);
int keypoint_transform(const float* kp, int n, double t00, double t02, double t11, double t12, int res, float* out, cudaStream_t st);
// the two above for several streams, one launch per pass (include/dynaboa_b200.h, "grouped input side"); every check but the
// NULL pointers of the C entries
int crop_resize_normalize_groups(const dboa_crop_desc* frames, int groups, unsigned long long active, int res, const float mean[3],
                                 const float stdv[3], float* tmp, long long tmp_floats, float* out, cudaStream_t st);
int keypoint_transform_groups(const float* kp, int n, const double* t4, int res, float* out, int groups, unsigned long long active,
                              cudaStream_t st);

// ---- eval.cu (evaluation metrics on the device)
size_t eval_scratch_floats(int B, int NJ);
int eval_metrics(const float* pred_verts, const float* gt_verts_joints, const float* gt_verts_pve, const float* Jreg, int NJ, int NV,
                 const int* joint_map, int n_map, float* scratch, float* out, int B, int groups, unsigned long long active, cudaStream_t st);

// render.cu: mesh overlay (include/dynaboa_b200.h, "mesh overlay")
long long render_scratch_bytes(int W, int H, int NV, int NF, int samples);
int render_overlay(const float* verts, const int* faces, const int* vf_offsets, const int* vf_faces, int NV, int NF, const float cam4[4],
                   const float rot3x3[9], const float color3[3], const unsigned char* img, int W, int H, int samples, void* scratch,
                   long long scratch_bytes, unsigned char* out, int* face_ids, cudaStream_t st);
long long render_scratch_bytes_groups(const int* W, const int* H, int M, int NV, int NF, int samples);
int render_overlay_groups(const dboa_render_desc* meshes, int M, const int* faces, const int* vf_offsets, const int* vf_faces, int NV,
                          int NF, int samples, void* scratch, long long scratch_bytes, cudaStream_t st);

}  // namespace dboa
