/* libdynaboa_b200 -- C ABI of the CUDA-native (H100, sm_90a) DynaBOA hot path.
 *
 * The reference (syguan96/DynaBOA) has no FFI/plugin boundary of its own: its hot path is Python
 * calling stock PyTorch ops (SURVEY.md §8b).  This header is the boundary the CUDA implementation
 * introduces underneath the reference's Python API; each entry point names the reference code it
 * replaces.  Conventions:
 *   - every pointer is a DEVICE pointer to fp32 data unless stated otherwise; buffers are owned by
 *     the caller (torch-allocated) and must outlive the call;
 *   - `stream` is a cudaStream_t passed as void*; kernels are enqueued on it and never synchronise;
 *   - return value: 0 = ok, <0 = error (DBOA_ERR_*); no exceptions cross the ABI;
 *   - one host thread per device (the reference is single-threaded on this path).
 * Reference-side binding (ctypes) is shown in INTEGRATION.md.
 */
#ifndef DYNABOA_B200_H
#define DYNABOA_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define DBOA_OK 0
#define DBOA_ERR_ARG (-1)
#define DBOA_ERR_SHAPE (-2)
#define DBOA_ERR_CUDA (-3)
#define DBOA_ERR_UNSUPPORTED (-4)

typedef void* dboa_stream_t;

/* ---- library state ------------------------------------------------------------------------- */
const char* dboa_version(void);
int dboa_last_cuda_error(void);            /* cudaError_t of the last failed launch */
long long dboa_launch_count(void);         /* kernels launched by this library so far */
/* add n >= 0 to dboa_launch_count: the kernels of a replayed CUDA graph, counted once when they were captured */
int dboa_launch_credit(long long n);
/* the one-time set-up of the network backward (side streams, events, device tables), made ahead of a CUDA graph capture; the
 * first eager backward makes it otherwise.  A library call that would still need set-up while its stream is being captured
 * returns DBOA_ERR_UNSUPPORTED and enqueues nothing. */
int dboa_prepare_graph(void);
/* cudaStreamWaitEvent(stream, event, cudaEventWaitExternal): captured into a graph, the wait applies on every replay to the
 * event's latest record made outside the graph (event: a cudaEvent_t) */
int dboa_stream_wait_external(dboa_stream_t stream, void* event);
/* which convolution products of the HMR plan run on the wgmma TF32x3 kernel -- 0: none (fp32 CUDA cores); 1: forward;
 * 2: forward + dgrad + wgrad; 3 (default, faster on H100 at batch 1): forward + dgrad, weight gradients on CUDA cores */
int dboa_set_tensor_core_conv(int mode);

/* 1: dboa_hmr_forward runs the fused plan -- every GroupNorm applied by the consuming convolution on load, its statistics
 * produced by the epilogue of the producing one (one convolution launch per layer); 0 (default, faster on H100): one
 * convolution and one GroupNorm launch per layer.  Both fill the same tape.  Environment: DBOA_FUSED_FWD. */
int dboa_set_fused_forward(int enable);
int dboa_get_fused_forward(void);
/* the same switch for dboa_hmr_backward: 1 = fused data-gradient chain (GroupNorm backward on load), 0 (default) =
 * GroupNorm-backward and data-gradient launches per layer.  Environment: DBOA_FUSED_BWD. */
int dboa_set_fused_backward(int enable);
int dboa_get_fused_backward(void);

/* ---- HMR regressor: parameter arena and tape layout ----------------------------------------
 * replaces: model/hmr.py:67-124 (HMR.__init__/_make_layer state_dict contract).
 * The 169 parameters live in ONE flat fp32 arena; entry i (in nn.Module.parameters() order) is the
 * strided view (offset, shape, stride) of it.  Conv weights are stored [Cout][kh][kw][Cin]. */
int dboa_hmr_num_params(void);
long long dboa_hmr_arena_floats(void);
int dboa_hmr_param_info(int i, char* name, int name_cap, long long* offset, int* ndim, long long shape[4], long long stride[4]);
long long dboa_hmr_tape_floats(int B);      /* activations saved by the forward (also holds the features) */
long long dboa_hmr_scratch_floats(int B);   /* scratch shared by forward (split-K) and backward */
/* Float offset of one region of the tape of batch B (host only, no device access), for tests and debugging tools that read
 * what the forward saved.  Per convolution `conv` (the conv whose weight is dboa_hmr_param_info(3 * conv)), NHWC:
 *   Y      (B,Ho,Wo,Cout) convolution output;  STATS (B,4,2) GroupNorm (mean, rstd) per (sample, group);
 *   A      (B,Ho,Wo,Cout) post-activation output -- DBOA_ERR_ARG for a downsample conv, whose block output is conv3's A.
 * Whole tape (`conv` ignored): X0 (B,224,224,3) image; P0 (B,56,56,64) max-pool output; P0_IDX the window position r*3+s of
 * each max-pool output as one byte, same (B,56,56,64) order; XC (3,B,2208) regressor input rows; H1PRE, H1POST, H2PRE, H2POST
 * (3,B,1024) hidden rows before / after dropout; PARAMS (4,B,160) running SMPL parameters (first 157 used); MASKS (3,2,B,1024)
 * dropout keep-masks.  Returns DBOA_ERR_SHAPE for B outside 1..64 and DBOA_ERR_ARG for an unknown kind or conv. */
#define DBOA_TAPE_Y 0
#define DBOA_TAPE_STATS 1
#define DBOA_TAPE_A 2
#define DBOA_TAPE_X0 3
#define DBOA_TAPE_P0 4
#define DBOA_TAPE_P0_IDX 5
#define DBOA_TAPE_XC 6
#define DBOA_TAPE_H1PRE 7
#define DBOA_TAPE_H1POST 8
#define DBOA_TAPE_H2PRE 9
#define DBOA_TAPE_H2POST 10
#define DBOA_TAPE_PARAMS 11
#define DBOA_TAPE_MASKS 12
long long dboa_hmr_tape_offset(int B, int kind, int conv);
/* feature i of HMR.forward(need_feature=True) (model/hmr.py:138-168) as a strided view of the tape */
int dboa_hmr_feature_info(int B, int i, long long* offset, int* ndim, long long shape[4], long long stride[4]);

/* replaces: model/hmr.py:127-181 HMR.forward (+ utils/geometry.py:47-61 rot6d_to_rotmat).
 * image: (B,3,224,224) NCHW.  drop_masks: NULL (eval) or (3,2,B,1024) keep-masks already scaled by 1/(1-p).
 * outputs: rotmat (B,24,3,3), shape (B,10), cam (B,3), pose6d (B,144). */
int dboa_hmr_forward(const float* arena, const float* init_pose, const float* init_shape, const float* init_cam,
                     const float* image, int B, const float* drop_masks, float* tape, float* scratch,
                     float* rotmat, float* shape, float* cam, float* pose6d, dboa_stream_t stream);
/* replaces: autograd backward of the above (torch.autograd.grad in learn2learn MAML.adapt, loss.backward()
 * at dynaboa_benchmark.py:140,150).  grad_arena is ACCUMULATED into (+=), same layout as the arena. */
int dboa_hmr_backward(const float* arena, const float* tape, int B, int masked /* forward used drop_masks */,
                      const float* d_rotmat, const float* d_shape, const float* d_cam, float* grad_arena, float* scratch,
                      dboa_stream_t stream);
/* Several independent videos in one launch sequence: the two calls above for `groups` videos of B / groups samples each.
 * Video g owns the consecutive samples [g * B / groups, (g + 1) * B / groups) of every per-sample buffer (image, masks, outputs,
 * d_* inputs; the tape and scratch are those of batch B) and the weights arena + g * dboa_hmr_arena_floats(); the backward
 * accumulates into grad_arena + g * dboa_hmr_arena_floats().  Each video's arithmetic is the single-video plan's (the split-K
 * slicing of a convolution may differ, since it is sized for all groups' tiles).  groups = 1 is exactly dboa_hmr_forward /
 * dboa_hmr_backward.  Checked before any device access: DBOA_ERR_SHAPE for groups < 1, B outside 1..64 or B % groups != 0;
 * DBOA_ERR_UNSUPPORTED for groups > 1 while the fused forward or backward plan is selected, and (backward) while
 * dboa_hmr_backward_buckets is armed.  A grouped backward call (groups != 1) always consumes an armed bucket request. */
int dboa_hmr_forward_groups(const float* arena, const float* init_pose, const float* init_shape, const float* init_cam,
                            const float* image, int B, const float* drop_masks, float* tape, float* scratch,
                            float* rotmat, float* shape, float* cam, float* pose6d, dboa_stream_t stream, int groups);
int dboa_hmr_backward_groups(const float* arena, const float* tape, int B, int masked, const float* d_rotmat,
                             const float* d_shape, const float* d_cam, float* grad_arena, float* scratch, dboa_stream_t stream,
                             int groups);
/* The two calls above with only some of the videos taking part: bit g of `active` set means video g is computed.  The grid,
 * split-K slicing and every other reduction split are those of the unmasked call, whose CTAs of idle videos return at once, so
 * each active video's outputs, tape rows and gradient are bit-identical to the unmasked call's.  An idle video's gradient arena
 * is not written; its rows of the outputs, tape and scratch are unspecified (nothing an active video computes reads them).
 * The _groups calls are these with every one of the `groups` bits set.  Checked before any device access, after the _groups
 * rules' DBOA_ERR_SHAPE: DBOA_ERR_ARG for active == 0 or a bit at position >= groups; then the _groups DBOA_ERR_UNSUPPORTED rules.
 * A masked backward call (groups != 1) always consumes an armed bucket request. */
int dboa_hmr_forward_active(const float* arena, const float* init_pose, const float* init_shape, const float* init_cam,
                            const float* image, int B, const float* drop_masks, float* tape, float* scratch,
                            float* rotmat, float* shape, float* cam, float* pose6d, dboa_stream_t stream, int groups,
                            unsigned long long active);
int dboa_hmr_backward_active(const float* arena, const float* tape, int B, int masked, const float* d_rotmat,
                             const float* d_shape, const float* d_cam, float* grad_arena, float* scratch, dboa_stream_t stream,
                             int groups, unsigned long long active);

/* Gradient buckets of the NEXT dboa_hmr_backward call, for overlapping the data-parallel all-reduce with the backward
 * (SURVEY.md section 8e).  Bucket k spans the floats [dboa_hmr_bucket_offset(k), dboa_hmr_bucket_offset(k - 1)) of the gradient
 * arena (offset(-1) = arena size): 0 = layer4 + regressor head, 1 = layer3, 2 = stem + layer1 + layer2 -- the order in which the
 * backward completes them.  ev0..2 are cudaEvent_t handles; event k is recorded when every kernel writing bucket k is ordered
 * before it.  Arm only for the LAST backward call that accumulates into the arena. */
int dboa_hmr_backward_buckets(void* ev0, void* ev1, void* ev2);
long long dboa_hmr_bucket_offset(int k);

/* ---- single operators (unit-parity surface; same kernels the plan above launches) ----------- */
/* replaces: nn.Conv2d forward / backward (model/hmr.py:29-34,72,113); NHWC activations, weights [Cout][Kpitch].
 * All three take Kpitch % 4 == 0 and Kpitch >= roundup16(k*k*Cin) (the weight rows are read / written as float4 up to the
 * next 16-element slab; the columns past k*k*Cin are zero padding the weight gradient leaves untouched), else DBOA_ERR_SHAPE;
 * the weight gradient of the 7x7 stem given a workspace (a kernel of its own) is held to the same rule.
 * forward: Cout % 64 == 0; data gradient: Cin % 64 == 0, Cout % 16 == 0; weight gradient: Cout % 64 == 0, dw accumulated (+=). */
int dboa_conv2d_fwd(const float* x, const float* w, float* y, int B, int Hi, int Wi, int Cin, int Cout, int k, int stride, int pad,
                    int Kpitch, float* ws, long long ws_floats, dboa_stream_t stream);
int dboa_conv2d_dgrad(const float* dy, const float* w, float* dx, int B, int Hi, int Wi, int Cin, int Cout, int k, int stride, int pad,
                      int Kpitch, int accumulate, float* ws, long long ws_floats, dboa_stream_t stream);
int dboa_conv2d_wgrad(const float* dy, const float* x, float* dw, int B, int Hi, int Wi, int Cin, int Cout, int k, int stride, int pad,
                      int Kpitch, float* ws, long long ws_floats, dboa_stream_t stream);
/* 1x1 / stride-1 convolution as a wgmma TF32x3 GEMM: y[M][Cout] = x[M][Cin] * w[Cout][Cin]^T (fp32-accurate);
 * needs dboa_set_tensor_core_conv(1); returns DBOA_ERR_UNSUPPORTED for shapes it does not take (Cin % 64, Cout % 64) */
int dboa_conv1x1_tc_fwd(const float* x, const float* w, float* y, int M, int Cin, int Cout, float* ws, long long ws_floats,
                        dboa_stream_t stream);
/* general convolution forward as a wgmma TF32x3 implicit GEMM (same arguments as dboa_conv2d_fwd; Cin % 64 == 0,
 * Cout % 64 == 0, Kpitch == k*k*Cin).  The stand-alone tensor-core entry points are launched with ordinary stream
 * serialization (inside dboa_hmr_forward/backward the same kernels use programmatic dependent launch and prefetch
 * weight tiles before their dependency wait, which needs the plan's guarantee that the preceding kernel does not write
 * the weights); DBOA_CABI_PDL=1 in the environment opts in for callers that can give that guarantee. */
int dboa_conv2d_tc_fwd(const float* x, const float* w, float* y, int B, int Hi, int Wi, int Cin, int Cout, int k, int stride, int pad,
                       int Kpitch, dboa_stream_t stream);
/* data / weight gradient on the same tensor-core kernel (needs dboa_set_tensor_core_conv(2 or 3)); dw is accumulated (+=) */
int dboa_conv2d_tc_dgrad(const float* dy, const float* w, float* dx, int B, int Hi, int Wi, int Cin, int Cout, int k, int stride, int pad,
                         int Kpitch, int accumulate, dboa_stream_t stream);
int dboa_conv2d_tc_wgrad(const float* dy, const float* x, float* dw, int B, int Hi, int Wi, int Cin, int Cout, int k, int stride, int pad,
                         int Kpitch, dboa_stream_t stream);
/* weight gradient on the wgmma tensor-core kernel whatever dboa_set_tensor_core_conv selects (csrc/conv_tc.cu): dw += dy^T *
 * im2col(x); Cin % 64 == 0, Cout % 64 == 0, Kpitch == k*k*Cin (DBOA_ERR_UNSUPPORTED otherwise) */
int dboa_conv2d_wgrad_tma(const float* dy, const float* x, float* dw, int B, int Hi, int Wi, int Cin, int Cout, int k, int stride, int pad,
                          int Kpitch, dboa_stream_t stream);
/* Fused convolution, the unit the forward plan is made of (csrc/conv_tc.cu: the operand transform runs in the loader).
 * replaces: nn.Conv2d + the nn.GroupNorm(4, C) / ReLU / residual add that PRECEDES it in Bottleneck.forward
 * (model/hmr.py:40-60), + the statistics pass of the GroupNorm that follows it.
 *   y = conv(T(x), w);  part_out[b][g] += (sum y, sum y^2) of group g of sample b, as 64-bit fixed point (scale 2^24):
 *   integer atomics, exact and order independent.  part_out (long long [B][4][2]) must be ZERO before the launch.
 *   mode 0: T(x) = x;  1: relu(gn(x));  2: relu(gn(x) + res);  3: relu(gn(x) + gn2(res))
 * gn statistics come from `part_in` (`part2_in`): the accumulators a previous call filled for x (res).
 * a_out / stats_out / stats2_out (optional): T(x) materialised, (mean, rstd) [B][4][2] of the GroupNorm(s).
 * Up to 2 problems per call (one launch each).  Cin % 64 == 0, Cout % 64 == 0, k in {1, 3}, stride 1 or 2 (DBOA_ERR_UNSUPPORTED otherwise). */
typedef struct dboa_fused_conv {
    const float *x, *res, *w;
    float *a_out, *stats_out, *stats2_out;
    const float *part_in, *part2_in, *gamma, *beta, *gamma2, *beta2;
    float *y, *part_out;
    int mode;
    int Hi, Cin, Cout, k, stride, pad;
} dboa_fused_conv;
long long dboa_conv_fused_part_floats(int B, int Ho, int Cout);   /* size of part_out in floats (= B * 16) */
int dboa_conv_fused_fwd(const dboa_fused_conv* probs, int nprob, int B, dboa_stream_t stream);

/* Fused data gradient, the unit the backward plan is made of (csrc/conv_tc.cu: GroupNorm backward in the loader).
 * replaces: the autograd backward of nn.GroupNorm (layer c) -> nn.Conv2d data gradient (layer c) -> residual add -> ReLU mask of
 * the producing layer p, + the reduction pass of GroupNorm_p's backward (model/hmr.py:40-60 under loss.backward()).
 *   dy  = rstd (dz gamma - m1 - x^ m2)                with (m1, m2) = sums_c / N, x^ = (y_c - mean) rstd     [dy_out: optional store]
 *   dX  = conv_c^T(dy) + addend                       stride 1, k in {1, 3}, Cin % 64 == 0, Cout % 64 == 0
 *   mask == NULL: out (+)= dX;   else out = dz_p = dX * (mask > 0) and, for each of the nprep GroupNorms of layer p,
 *   prep_sums[j][b][g] += (sum q, sum q x^), prep_dgb[j][c] += (d gamma, d beta) as 64-bit fixed point (scale 2^28; long long
 *   buffers the caller zeroes; integer atomics: exact and order independent). */
typedef struct dboa_dgrad_args {
    const float *dz, *y_c, *w, *stats_c, *sums_c, *gamma_c;
    float* dy_out;
    const float* addend;
    float* out;
    const float* mask;
    const float *prep_y[2], *prep_stats[2], *prep_gamma[2];
    float *prep_sums[2], *prep_dgb[2];
    int nprep, accumulate;
} dboa_dgrad_args;
int dboa_dgrad_fused(const dboa_dgrad_args* f, int B, int H, int Cin, int Cout, int k, dboa_stream_t stream);

/* replaces: nn.GroupNorm(4, C) + ReLU (+ residual) forward / backward (model/hmr.py:14-18,40-60).
 * C / 16 must be a power of two; one launch each (thread-block clusters).  `partial` is caller-provided scratch of
 * dboa_gn_*partial_floats() floats; the forward size is 0 in this version and the pointer may then be NULL. */
long long dboa_gn_partial_floats(int B, int HW, int C);
long long dboa_gn_bwd_partial_floats(int B, int HW, int C);
int dboa_groupnorm_fwd(const float* y, const float* gamma, const float* beta, const float* residual, float* out, float* stats,
                       float* partial, int B, int HW, int C, int relu, dboa_stream_t stream);
/* dgamma / dbeta are accumulated (+=).  With B > 1 the last cluster to finish sums the per-sample rows in sample order; it
 * is found through ticket counters the library holds once per process, so two such calls must not run concurrently (on
 * two streams): calls ordered on one stream are fine. */
int dboa_groupnorm_bwd(const float* dout, const float* mask_src, const float* y, const float* stats, const float* gamma, float* dy,
                       float* dgamma, float* dbeta, float* partial, int B, int HW, int C, dboa_stream_t stream);
/* replaces: nn.MaxPool2d(3, 2, 1) (model/hmr.py:75) on NHWC; idx holds each output's window position r * 3 + s (first maximum
 * in scan order, NaN propagates).  H and W even (output H/2 x W/2) and C % 4 == 0, else DBOA_ERR_SHAPE. */
int dboa_maxpool_fwd(const float* x, float* y, unsigned char* idx, int B, int H, int W, int C, dboa_stream_t stream);
int dboa_maxpool_bwd(const float* dy, const unsigned char* idx, float* dx, int B, int H, int W, int C, dboa_stream_t stream);

/* ---- rotations (utils/geometry.py) ---------------------------------------------------------- */
int dboa_rot6d_fwd(const float* x6, float* R, int n, dboa_stream_t stream);                       /* :47-61 */
int dboa_rot6d_bwd(const float* x6, const float* dR, float* dx6, int n, dboa_stream_t stream);
/* kind 0: batch_rodrigues :9-45 (quaternion route); kind 1: smplx lbs.batch_rodrigues (pose2rot=True) */
int dboa_rodrigues(const float* aa, float* R, int n, int kind, dboa_stream_t stream);
int dboa_rotmat_to_aa_fwd(const float* R, float* aa, int n, dboa_stream_t stream);              /* :184-306 */
int dboa_rotmat_to_aa_bwd(const float* R, const float* daa, float* dR, int n, dboa_stream_t stream);

/* ---- SMPL (model/smpl.py:25-37 over smplx lbs) ---------------------------------------------- */
typedef struct dboa_smpl_model {
    const float* v_template;   /* (6890,3) */
    const float* blend_dirs;   /* (217, 20670): rows 0..9 shapedirs as (l, v*3+k), rows 10..216 posedirs */
    const float* J_template;   /* (24,3)   = J_regressor @ v_template */
    const float* J_shapedirs;  /* (24,3,10) = J_regressor @ shapedirs */
    const int* parents;        /* (24,) */
    const float* lbs_weights;  /* (6890,24) */
    const float* J_extra;      /* (9,6890) reference config.JOINT_REGRESSOR_TRAIN_EXTRA */
    const int* joint_map;      /* (49,) into [24 kinematic | 21 vertex picks | 9 extra] */
    const int* vertex_ids;     /* (21,) smplx vertex_joint_selector picks */
} dboa_smpl_model;
long long dboa_smpl_tape_floats(int B);
long long dboa_smpl_scratch_floats(int B);
/* betas (B,10), rotmat (B,24,3,3) -> vertices (B,6890,3), joints (B,49,3) */
int dboa_smpl_forward(const dboa_smpl_model* m, const float* betas, const float* rotmat, int B, float* vertices, float* joints,
                      float* tape, dboa_stream_t stream);
/* d(joints) -> d(rotmat), d(betas) (vertices carry no loss on the adaptation path: SURVEY.md Appendix A) */
int dboa_smpl_backward(const dboa_smpl_model* m, const float* rotmat, int B, const float* tape, const float* d_joints, float* scratch,
                       float* d_rotmat, float* d_betas, int accumulate, dboa_stream_t stream);

/* ---- projection and losses (base_adaptor.py) ------------------------------------------------ */
int dboa_project_fwd(const float* cam, const float* j3d, float* p2d, int B, int NJ, dboa_stream_t stream);      /* :160-170 */
int dboa_project_bwd(const float* cam, const float* j3d, const float* dp2d, float* dj3d, float* dcam, int B, int NJ, int acc_j,
                     int acc_cam, dboa_stream_t stream);
/* GMM pose prior (:405-409, utils/smplify/prior.py:181-196): prior_b[b] = min_m NLL; d_rotmat = scale * d prior_b / dR */
int dboa_pose_prior(const float* rotmat, const float* means, const float* precisions, const float* neg_log_w, float* prior_b,
                    float* d_rotmat, float scale, int B, dboa_stream_t stream);
/* MaxMixturePrior.forward(pose, betas) itself (utils/smplify/prior.py:227-231) on a (B,69) axis-angle body pose */
int dboa_gmm_prior(const float* pose69, const float* means, const float* precisions, const float* neg_log_w, float* prior_b,
                   float* d_pose, float scale, int B, dboa_stream_t stream);
typedef struct dboa_loss_args {
    int B;
    const float *p2d, *j3d, *R, *beta;      /* predictions: (B,49,2) (B,49,3) (B,24,3,3) (B,10) */
    const float* kp;                        /* (B,49,3) keypoints + confidence, or NULL */
    const float* prior_b;                   /* (B,) per-body pose prior values, or NULL */
    const float *t_p2d, *t_j3d, *t_beta, *t_R; /* consistency / label targets, or NULL each */
    const float* gt_s3d;                    /* (B,24,4) labelled 3D joints, or NULL (needs kp) */
    float w[8];                             /* weights: s2d, shape, pose, t_p2d, t_j3d, t_beta, t_R, s3d */
    float* terms;                           /* (9,) out: the 8 unweighted terms, then the weighted total */
    float *dp2d, *dj3d, *dR, *dbeta;        /* out: gradients of the weighted total (NULL to skip) */
    int dR_accumulate;                      /* 1: dR already holds the pose-prior gradient */
    int kp_first, kp_count;                 /* joints [kp_first, kp_first + kp_count) of the 49 carry the 2D re-projection term; 0, 0 = the
                                               benchmark's 24 ground-truth joints (25, 24); the webcam client compares the 25 OpenPose
                                               joints (0, 25), reference dynaboa_webcam.py:236,246,262 */
    int groups;                             /* 0 or 1: one learner.  G > 1: B = G * b rows of G independent videos (video g: rows
                                               [g b, (g+1) b) of every per-row buffer); means, gradient scaling and prior_b sums are
                                               per video and `terms` is (G, 9).  B % G must be 0 */
} dboa_loss_args;
int dboa_loss_multi(const dboa_loss_args* args, dboa_stream_t stream);        /* :234-241,283-291,331-337,360-370,401,412-422 */
int dboa_loss_motion(const float* p_cur, const float* p_hist, const float* kp_cur, const float* kp_hist, float weight, float* term,
                     float* dp_cur, float* dp_hist, int B, int accumulate_cur, dboa_stream_t stream);               /* :379-398 */
/* the same on joints [first, first + count): reference dynaboa_webcam.py:161-181 uses the 25 OpenPose joints (0, 25) */
int dboa_loss_motion_joints(const float* p_cur, const float* p_hist, const float* kp_cur, const float* kp_hist, float weight, float* term,
                            float* dp_cur, float* dp_hist, int B, int accumulate_cur, int first, int count, dboa_stream_t stream);
/* the same for `groups` independent videos of B / groups rows each: the mean is per video and term is (groups,) */
int dboa_loss_motion_groups(const float* p_cur, const float* p_hist, const float* kp_cur, const float* kp_hist, float weight, float* term,
                            float* dp_cur, float* dp_hist, int B, int accumulate_cur, int first, int count, int groups,
                            dboa_stream_t stream);
/* the same with a per-video enable: a video whose `active` bit is clear gets term[g] = 0 and leaves its rows of dp_cur and
 * dp_hist untouched.  DBOA_ERR_SHAPE for groups outside 1..64 or B % groups != 0, DBOA_ERR_ARG for active == 0 or a bit at
 * position >= groups */
int dboa_loss_motion_active(const float* p_cur, const float* p_hist, const float* kp_cur, const float* kp_hist, float weight, float* term,
                            float* dp_cur, float* dp_hist, int B, int accumulate_cur, int first, int count, int groups,
                            unsigned long long active, dboa_stream_t stream);

/* ---- per-video hyperparameters ---------------------------------------------------------------
 * The calls below give each of `groups` (1..64) videos its own scalars, in the layout of the grouped calls above: video g owns
 * the rows [g B / groups, (g + 1) B / groups) of every per-row buffer (and, in the sweeps further down, the floats
 * [g n, (g + 1) n) of every arena).  The per-video scalars are HOST arrays with one row per video; they travel in the launch
 * parameters, so no device table is allocated and a captured call holds its values.  Video g's outputs are bit-identical to
 * the uniform call on its rows with its row of scalars (each entry the fp32 value the uniform call receives).  Checked before any
 * device access: DBOA_ERR_ARG for a NULL pointer or table, DBOA_ERR_SHAPE for groups outside 1..64 or B % groups != 0, then
 * (calls with `active`) DBOA_ERR_ARG for active == 0 or a bit at position >= groups.
 * dboa_pose_prior_groups: dboa_pose_prior with scale (groups,): body b's gradient is scaled by scale[b / (B / groups)]. */
int dboa_pose_prior_groups(const float* rotmat, const float* means, const float* precisions, const float* neg_log_w, float* prior_b,
                           float* d_rotmat, const float* scale, int B, int groups, dboa_stream_t stream);
/* dboa_loss_multi with w (a->groups, 8): video g's block uses row g in place of a->w (a->w is not read); the other arguments
 * and their checks are dboa_loss_multi's */
int dboa_loss_multi_weights(const dboa_loss_args* a, const float* w, dboa_stream_t stream);
/* dboa_loss_motion_active with weight (groups,): video g's gradient is weighed with weight[g]; a video whose bit is clear gets
 * term[g] = 0 and leaves its rows of dp_cur and dp_hist untouched, as there */
int dboa_loss_motion_weights(const float* p_cur, const float* p_hist, const float* kp_cur, const float* kp_hist, const float* weight,
                             float* term, float* dp_cur, float* dp_hist, int B, int accumulate_cur, int first, int count, int groups,
                             unsigned long long active, dboa_stream_t stream);

/* ---- whole-model sweeps, feature test, retrieval -------------------------------------------- */
int dboa_sgd_update(const float* p, const float* g, float* out, float lr, long long n, dboa_stream_t stream);   /* l2l maml_update */
/* Adam + EMA teacher (base_adaptor.py:126,193-201) with the arithmetic of torch's single-tensor Adam: the fp32 scalars of
 * the sweep (1 - beta1, beta2, 1 - beta2, the bias corrections, the step size, eps, alpha, 1 - alpha) are derived from
 * these double hyperparameters and each rounded once, as torch derives them from Python floats */
int dboa_adam_ema(float* p, const float* g, float* m, float* v, float* teacher /* or NULL */, long long n, double lr, double beta1,
                  double beta2, double eps, int step, double alpha, dboa_stream_t stream);
int dboa_ema_update(float* teacher, const float* p, long long n, double alpha, dboa_stream_t stream);
/* Adam(+EMA) on g * gscale: the data-parallel mean of an all-reduced (summed) gradient without a separate sweep */
int dboa_adam_ema_scaled(float* p, const float* g, float* m, float* v, float* teacher /* or NULL */, long long n, double lr, double beta1,
                         double beta2, double eps, int step, double alpha, float gscale, dboa_stream_t stream);
/* the DBOA_ADAM_SCALARS fp32 scalars of one dboa_adam_ema_scaled sweep, derived on the host as it derives them, into the host
 * array out: 1 - beta1, beta2, 1 - beta2, sqrt(bias correction 2), eps, -(lr / bias correction 1), alpha, 1 - alpha, gscale */
#define DBOA_ADAM_SCALARS 9
int dboa_adam_scalars(float* out, double lr, double beta1, double beta2, double eps, int step, double alpha, float gscale);
/* dboa_adam_ema_scaled with its scalars read from the device block `scalars` (dboa_adam_scalars' order) when the kernel runs:
 * a sweep captured into a CUDA graph takes the step's bias correction from the block, written before each replay; same
 * arithmetic, bit for bit */
int dboa_adam_ema_dev(float* p, const float* g, float* m, float* v, float* teacher /* or NULL */, long long n, const float* scalars,
                      dboa_stream_t stream);
/* Per-video sweeps (see "per-video hyperparameters" above): `groups` arenas of n floats each (n % 4 == 0, else
 * DBOA_ERR_SHAPE), of which only the videos whose bit is set in `active` take part -- the floats of the others are neither read
 * nor written, and the grid covers the active videos only.  dboa_sgd_update_groups: lr (groups,), video g's step is
 * dboa_sgd_update with lr[g].  dboa_adam_ema_groups: scalars (groups, DBOA_ADAM_SCALARS), row g written by dboa_adam_scalars
 * from video g's lr, betas, eps, step count and alpha; video g's sweep is dboa_adam_ema_dev with that row, so active videos at
 * different step counts share one launch. */
int dboa_sgd_update_groups(const float* p, const float* g, float* out, const float* lr, long long n, int groups, unsigned long long active,
                           dboa_stream_t stream);
int dboa_adam_ema_groups(float* p, const float* g, float* m, float* v, float* teacher /* or NULL */, long long n, const float* scalars,
                         int groups, unsigned long long active, dboa_stream_t stream);
/* stream-ordered fill / device-to-device copy on the copy engine (gradient arenas, frame staging: no ATen kernels in a step) */
int dboa_fill_zero(void* dst, long long bytes, dboa_stream_t stream);
int dboa_copy_async(void* dst, const void* src, long long bytes, dboa_stream_t stream);
/* cal_feature_diff :211-219: cosine similarity of npairs (<=16) flattened tensor pairs; host arrays of device pointers */
int dboa_cosine_pairs(const float* const* a, const float* const* b, const long long* n, int npairs, float* partial,
                      long long partial_floats, float* out, float eps, dboa_stream_t stream);
/* the same reduction, returning per pair the three sums (a.b, |a|^2, |b|^2) in double, [npairs][3]: under data-parallel
 * adaptation they are all-reduced before the cosine is formed, so that every rank takes the same branch of the
 * dynamic loop (dynaboa_benchmark.py:161-192; cal_feature_diff flattens across the batch, base_adaptor.py:215).
 * partial: dboa_cosine_partial_floats(n, npairs) floats of scratch. */
long long dboa_cosine_partial_floats(const long long* n, int npairs);
int dboa_cosine_terms(const float* const* a, const float* const* b, const long long* n, int npairs, float* partial,
                      long long partial_floats, double* terms, dboa_stream_t stream);
/* the same for `groups` videos at once, each on its own part of every pair: the per-video feature test of the dynamic loop
 * of MultiVideoAdaptor.  n[i] is the length of pair i over all groups; video g's part is the floats
 * [g n[i] / groups, (g + 1) n[i] / groups) of a[i] and b[i] (the per-sample layout of every dboa_hmr_feature_info view, made
 * dense).  terms: [groups][npairs][3] in double.  Only the videos whose bit is set in `active` take part: the rows of terms of
 * the others are not written and none of their inputs is read.  Video g's sums are bit-identical to dboa_cosine_terms on its
 * parts alone; groups = 1 with bit 0 set is dboa_cosine_terms.  partial: dboa_cosine_partial_floats_groups(n, npairs, groups)
 * floats of scratch.  DBOA_ERR_ARG for a NULL pointer, npairs outside 1..16, active == 0, a bit at position >= groups or too
 * small a partial; DBOA_ERR_SHAPE for groups outside 1..64 or n[i] % groups != 0 (both the same for the floats query). */
long long dboa_cosine_partial_floats_groups(const long long* n, int npairs, int groups);
int dboa_cosine_terms_active(const float* const* a, const float* const* b, const long long* n, int npairs, float* partial,
                             long long partial_floats, double* terms, dboa_stream_t stream, int groups, unsigned long long active);
/* retrieval :82-84: index of the centre with the smallest cosine distance to feat (D,) among centers (K,D) */
int dboa_retrieval_nearest(const float* feat, const float* centers, int K, int D, int* best, float* dists, dboa_stream_t stream);

/* ---- input side: crop + resize + normalise, keypoint transform (utils/dataprocess.py:13-96, boa_dataset/pw3d.py:127-163) ---
 * img: device image (H,W,3) RGB, float32 0..255 or uint8 (is_u8).  The crop box [ul, ul + (Wc, Hc)) (integer corners as the
 * reference computes them; zero outside the frame) is resized to res x res as  out = Wy . crop . Wx^T : wx (res,Tx) / wy (res,Ty)
 * are the rows of the banded matrices (skimage.transform.resize = Gaussian pre-filter + order-1 zoom, mirror boundaries,
 * composed on the host), sx / sy (res,) int32 their first crop column / row.  Host arrays mean3 / std3: channel statistics.
 * tmp: Hc * res * 3 floats of scratch.  out: (3,res,res) = (resized / 255 - mean) / std. */
int dboa_crop_resize_normalize(const void* img, int is_u8, int H, int W, int ul_x, int ul_y, int Hc, const float* wx, const int* sx, int Tx,
                               const float* wy, const int* sy, int Ty, int res, const float* mean3, const float* std3, float* tmp,
                               float* out, dboa_stream_t stream);
/* kp (n,3) pixel keypoints + confidence -> out (n,3): p = trunc(t . (x, y, 1)) + 1 in double as utils/dataprocess.py:39-46 on kp + 1,
 * then 2 p / res - 1; t00, t02, t11, t12: the non-zero entries of get_transform(center, scale, res) (:13-37, rot = 0) */
int dboa_keypoint_transform(const float* kp, int n, double t00, double t02, double t11, double t12, int res, float* out,
                            dboa_stream_t stream);
/* Grouped input side: the two calls above for the frames of `groups` streams (one camera each), of which those whose bit is
 * set in `active` take part.  One frame per stream; frames may differ in size and dtype.  dboa_crop_desc: the arguments of
 * dboa_crop_resize_normalize that describe one frame and its crop (img, is_u8, H, W, ul_x, ul_y, Hc and the wx / sx / Tx,
 * wy / sy / Ty tables, all device pointers).  `frames` is a HOST array of `groups` descriptors; the active ones are passed to
 * the kernels by value, so a call makes no host-to-device copy and never synchronises (the descriptors of idle streams are
 * not read).  Two launches, whatever `groups`: the rows pass over every active frame's Hc * res outputs, then one grid row per
 * active frame.  tmp: sum over the active frames of Hc * res * 3 floats (tmp_floats: its size).  out (groups,3,res,res): row g
 * of an active stream is bit-identical to dboa_crop_resize_normalize on frame g alone; the frames of idle streams are not
 * read and their rows of out are not written.
 * Before any device access: DBOA_ERR_ARG for a NULL frames, mean3, std3, tmp or out, DBOA_ERR_SHAPE for groups
 * outside 1..64 or res < 1, DBOA_ERR_ARG for active == 0 or a bit at position >= groups, then, per active descriptor,
 * DBOA_ERR_ARG for a NULL pointer and DBOA_ERR_SHAPE for H, W, Hc, Tx or Ty < 1, then DBOA_ERR_ARG for too small a tmp. */
typedef struct dboa_crop_desc {
    const void* img;
    const float* wx;
    const int* sx;
    const float* wy;
    const int* sy;
    int is_u8, H, W, ul_x, ul_y, Hc, Tx, Ty;
} dboa_crop_desc;
int dboa_crop_resize_normalize_groups(const dboa_crop_desc* frames, int groups, unsigned long long active, int res, const float* mean3,
                                      const float* std3, float* tmp, long long tmp_floats, float* out, dboa_stream_t stream);
/* kp (groups,n,3) detections of every stream -> rows [0, n) of out (groups,49,3) as dboa_keypoint_transform (bit for bit), rows
 * [n, 49) zeroed; t4: HOST array (groups,4) of each stream's t00, t02, t11, t12.  Streams whose bit is clear in `active`: kp
 * not read, out not written.  DBOA_ERR_ARG for a NULL pointer, DBOA_ERR_SHAPE for groups outside 1..64, n outside 0..49 or
 * res < 1, then DBOA_ERR_ARG for active == 0 or a bit at position >= groups; all before any device access.  One launch. */
int dboa_keypoint_transform_groups(const float* kp, int n, const double* t4, int res, float* out, int groups, unsigned long long active,
                                   dboa_stream_t stream);

/* ---- evaluation metrics (dynaboa_benchmark.py:217-240, utils/pose_utils.py:9-64) -----------------
 * pred_verts, gt_verts_joints (gender-selected SMPL mesh), gt_verts_pve (neutral mesh): (B,NV,3);
 * J_regressor (NJ,NV) dense; joint_map (n_map,) int32 indices into the NJ regressed joints (H36M_TO_J14).
 * Joints are centred on regressed joint 0 (pelvis) like the reference.  out (B,3) = MPJPE, PA-MPJPE (similarity
 * Procrustes, 3x3 SVD on the device) and PVE per sample, in the unit of the meshes (metres).
 * scratch: dboa_eval_scratch_floats(B, NJ) floats.  NJ, n_map <= 32. */
long long dboa_eval_scratch_floats(int B, int NJ);
int dboa_eval_metrics(const float* pred_verts, const float* gt_verts_joints, const float* gt_verts_pve, const float* J_regressor, int NJ,
                      int NV, const int* joint_map, int n_map, float* scratch, float* out, int B, dboa_stream_t stream);
/* the same for `groups` videos of b = B / groups rows each (video g owns the rows [g b, (g + 1) b)), of which only the videos
 * whose bit is set in `active` take part: the rows of the others are not read and their rows of out are not written.  An
 * active row is bit-identical to dboa_eval_metrics on that video's rows alone; groups = 1 with bit 0 set is dboa_eval_metrics.
 * Before any device access: DBOA_ERR_ARG for a NULL pointer, DBOA_ERR_SHAPE for NJ or n_map outside 1..32, B < 1, groups
 * outside 1..64 or B % groups != 0, then DBOA_ERR_ARG for active == 0 or a bit at position >= groups. */
int dboa_eval_metrics_active(const float* pred_verts, const float* gt_verts_joints, const float* gt_verts_pve, const float* J_regressor,
                             int NJ, int NV, const int* joint_map, int n_map, float* scratch, float* out, int B, int groups,
                             unsigned long long active, dboa_stream_t stream);

/* ---- mesh overlay (render_demo.py:58-153) -----------------------------------------------------
 * replaces: Renderer.render (pyrender + trimesh, OpenGL off-screen) as called by base_adaptor.py:429-443 and
 * utils/webcam_utils.py:71-79.  Draws one mesh over one frame; the contract (camera, culling, fill rule, depth, sample
 * pattern, shading, composite) is DESIGN.md section 6 "Mesh overlay" and the header of csrc/render.cu.
 * verts (NV,3) fp32, faces (NF,3) int32; vf_offsets (NV+1) / vf_faces (3 NF) int32: the vertex->face adjacency (CSR, faces
 * of each vertex in ascending order), built once per faces array.  Host arrays: cam4 = (sx, sy, tx, ty) in the frame
 * (convert_crop_cam_to_orig_img :136-153), rot3x3 = row-major angle/axis rotation applied after Rx(180) (NULL: none),
 * color3 = base colour (0..1).  img / out (H,W,3) uint8 (channels pass through in the order given); face_ids (H,W,samples)
 * int32 = winning face per sample, -1 where nothing is covered (NULL: not written).  samples 1 or 4.
 * scratch: dboa_render_scratch_bytes() bytes.  W, H <= 8192, NV, NF >= 0 (DBOA_ERR_SHAPE otherwise).  Two calls on the same
 * inputs give bit-identical out and face_ids. */
long long dboa_render_scratch_bytes(int W, int H, int NV, int NF, int samples);
int dboa_render_overlay(const float* verts, const int* faces, const int* vf_offsets, const int* vf_faces, int NV, int NF, const float cam4[4],
                        const float rot3x3[9], const float color3[3], const unsigned char* img, int W, int H, int samples, void* scratch,
                        long long scratch_bytes, unsigned char* out, int* face_ids, dboa_stream_t stream);
/* Grouped overlay: M meshes of one topology (faces, vf_offsets, vf_faces, NV, NF) and one sample count, each over its own
 * frame, in one call: the adapted and the base mesh of every webcam stream of a tick.  dboa_render_desc: the per-mesh
 * arguments of dboa_render_overlay (verts, img, out and face_ids are device pointers, face_ids may be NULL; has_rot = 0
 * means no rotation and rot3x3 is not read; W, H the frame size of that mesh).  `meshes` is a HOST array of M descriptors,
 * passed to the kernels by value, so a call makes no host-to-device copy and never synchronises.  Two entries may read the
 * same img; the outputs (out, face_ids) must not alias any input or each other.  6 kernel launches and 1 memset, whatever M:
 * vertices, normals and face set-up take the mesh from the grid's y index, the scan runs one block per mesh, the raster walks
 * the (mesh, face, tile) pairs of all meshes, the resolve gives every mesh its own row blocks.  Every mesh's out and face_ids
 * are bit-identical to dboa_render_overlay on that entry alone; M = 1 is dboa_render_overlay.
 * scratch: dboa_render_scratch_bytes_groups(W, H, M, NV, NF, samples) bytes (W, H: host arrays of the M frame sizes; M = 1
 * gives dboa_render_scratch_bytes).  Before any device access: DBOA_ERR_ARG for a NULL meshes, faces, vf_offsets, vf_faces or
 * scratch; DBOA_ERR_SHAPE for M outside 1..64, NV or NF < 0 or any W or H outside 1..8192; then DBOA_ERR_ARG for samples
 * other than 1 or 4, an entry's NULL verts, img or out, or too small a scratch.  The size query returns the same codes. */
typedef struct dboa_render_desc {
    const float* verts;
    const unsigned char* img;
    unsigned char* out;
    int* face_ids;
    float cam4[4];
    float rot3x3[9];
    int has_rot;
    float color3[3];
    int W, H;
} dboa_render_desc;
long long dboa_render_scratch_bytes_groups(const int* W, const int* H, int M, int NV, int NF, int samples);
int dboa_render_overlay_groups(const dboa_render_desc* meshes, int M, const int* faces, const int* vf_offsets, const int* vf_faces, int NV,
                               int NF, int samples, void* scratch, long long scratch_bytes, dboa_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DYNABOA_B200_H */
