// Whole-network launch plan of the HMR regressor: parameter arena layout, activation tape layout,
// forward and hand-written backward (no autograd-through-autograd).
//
// Replaces reference model/hmr.py:67-124 (module construction / state_dict contract),
// :127-181 (HMR.forward, Bottleneck.forward :40-60) and the torch autograd backward that
// learn2learn's MAML.adapt / loss.backward() run over it (reference dynaboa_benchmark.py:140,150).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.h"
#include "../../include/dynaboa_b200.h"

namespace dboa {

int g_last_cuda_error = 0;
long long g_launch_count = 0;
bool pdl_enabled() {
    static const bool on = [] { const char* e = getenv("DBOA_PDL"); return !(e && e[0] == '0'); }();
    return on;
}

// ---------------------------------------------------------------------------------------------
// static network description
// ---------------------------------------------------------------------------------------------
struct ConvLayer {
    std::string wname, nname;      // state_dict prefixes of the conv and its GroupNorm
    int cin, cout, k, stride, pad, hin, hout, kpitch;
    long long w_off, g_off, b_off; // arena offsets (floats)
};
struct Block { int c1, c2, c3, cd; };     // conv indices; cd = -1 when the residual is the identity

struct ParamInfo { std::string name; long long off; int ndim; long long shape[4], stride[4]; };

struct Net {
    std::vector<ConvLayer> convs;
    std::vector<Block> blocks;
    std::vector<ParamInfo> params;       // nn.Module.parameters() order of the reference
    long long arena_floats = 0;
    long long fc1_w, fc1_b, fc2_w, fc2_b, dec_w, dec_b;
};

static long long align32(long long x) { return (x + 31) / 32 * 32; }

static const int kBlocks[4] = {3, 4, 6, 3}, kPlanes[4] = {64, 128, 256, 512};
static const int HEAD_IN = 2205, HEAD_LD = 2208, HID = 1024, NDEC = 157, DEC_LD = 160;

static Net build_net() {
    Net n;
    long long off = 0;
    auto add_conv = [&](const std::string& wname, const std::string& nname, int cin, int cout, int k, int stride, int pad, int hin) {
        ConvLayer c;
        c.wname = wname; c.nname = nname; c.cin = cin; c.cout = cout; c.k = k; c.stride = stride; c.pad = pad; c.hin = hin;
        c.hout = (hin + 2 * pad - k) / stride + 1;
        int K = k * k * cin;
        c.kpitch = (K + 15) / 16 * 16;
        c.w_off = off; off = align32(off + (long long)cout * c.kpitch);
        c.g_off = off; off = align32(off + cout);
        c.b_off = off; off = align32(off + cout);
        ParamInfo w{wname + ".weight", c.w_off, 4, {cout, cin, k, k}, {c.kpitch, 1, (long long)k * cin, cin}};
        ParamInfo g{nname + ".weight", c.g_off, 1, {cout, 1, 1, 1}, {1, 1, 1, 1}};
        ParamInfo b{nname + ".bias", c.b_off, 1, {cout, 1, 1, 1}, {1, 1, 1, 1}};
        n.params.push_back(w); n.params.push_back(g); n.params.push_back(b);
        n.convs.push_back(c);
        return (int)n.convs.size() - 1;
    };
    add_conv("conv1", "bn1", 3, 64, 7, 2, 3, 224);
    int inpl = 64, h = 56;
    for (int li = 0; li < 4; ++li) {
        for (int bi = 0; bi < kBlocks[li]; ++bi) {
            int s = (li > 0 && bi == 0) ? 2 : 1, pl = kPlanes[li];
            char pre[64];
            snprintf(pre, sizeof pre, "layer%d.%d", li + 1, bi);
            Block b;
            b.c1 = add_conv(std::string(pre) + ".conv1", std::string(pre) + ".bn1", inpl, pl, 1, 1, 0, h);
            b.c2 = add_conv(std::string(pre) + ".conv2", std::string(pre) + ".bn2", pl, pl, 3, s, 1, h);
            int hout = h / s;
            b.c3 = add_conv(std::string(pre) + ".conv3", std::string(pre) + ".bn3", pl, pl * 4, 1, 1, 0, hout);
            b.cd = -1;
            if (bi == 0) b.cd = add_conv(std::string(pre) + ".downsample.0", std::string(pre) + ".downsample.1", inpl, pl * 4, 1, s, 0, h);
            n.blocks.push_back(b);
            inpl = pl * 4; h = hout;
        }
    }
    n.fc1_w = off; off = align32(off + (long long)HID * HEAD_LD);
    n.fc1_b = off; off = align32(off + HID);
    n.fc2_w = off; off = align32(off + (long long)HID * HID);
    n.fc2_b = off; off = align32(off + HID);
    n.dec_w = off; off = align32(off + (long long)NDEC * HID);
    n.dec_b = off; off = align32(off + NDEC);
    n.params.push_back({"fc1.weight", n.fc1_w, 2, {HID, HEAD_IN, 1, 1}, {HEAD_LD, 1, 1, 1}});
    n.params.push_back({"fc1.bias", n.fc1_b, 1, {HID, 1, 1, 1}, {1, 1, 1, 1}});
    n.params.push_back({"fc2.weight", n.fc2_w, 2, {HID, HID, 1, 1}, {HID, 1, 1, 1}});
    n.params.push_back({"fc2.bias", n.fc2_b, 1, {HID, 1, 1, 1}, {1, 1, 1, 1}});
    n.params.push_back({"decpose.weight", n.dec_w, 2, {144, HID, 1, 1}, {HID, 1, 1, 1}});
    n.params.push_back({"decpose.bias", n.dec_b, 1, {144, 1, 1, 1}, {1, 1, 1, 1}});
    n.params.push_back({"decshape.weight", n.dec_w + 144LL * HID, 2, {10, HID, 1, 1}, {HID, 1, 1, 1}});
    n.params.push_back({"decshape.bias", n.dec_b + 144, 1, {10, 1, 1, 1}, {1, 1, 1, 1}});
    n.params.push_back({"deccam.weight", n.dec_w + 154LL * HID, 2, {3, HID, 1, 1}, {HID, 1, 1, 1}});
    n.params.push_back({"deccam.bias", n.dec_b + 154, 1, {3, 1, 1, 1}, {1, 1, 1, 1}});
    n.arena_floats = off;
    return n;
}

static const Net& net() {
    static Net n = build_net();
    return n;
}

// ---------------------------------------------------------------------------------------------
// activation tape
// ---------------------------------------------------------------------------------------------
struct ConvTape { long long y, part, stats, a; };   // a == -1: output lives in the block's conv3 slot
struct Tape {
    long long x0, p0, p0_idx;
    long long acc;                  // fixed-point GroupNorm statistics of the fused plan: long long [conv][B][4][2]
    std::vector<ConvTape> conv;
    long long xc, h1pre, h1post, h2pre, h2post, params, masks;
    long long total;
};

static Tape build_tape(int B) {
    const Net& n = net();
    Tape t;
    long long off = 0;
    auto take = [&](long long cnt) { long long o = off; off = align32(off + cnt); return o; };
    t.x0 = take((long long)B * 224 * 224 * 3);
    t.conv.resize(n.convs.size());
    for (size_t i = 0; i < n.convs.size(); ++i) {
        const ConvLayer& c = n.convs[i];
        long long sz = (long long)B * c.hout * c.hout * c.cout;
        t.conv[i].y = take(sz);
        t.conv[i].part = take((long long)gn_partial_floats(B, c.hout * c.hout, c.cout));
        t.conv[i].stats = take((long long)B * 8);
        t.conv[i].a = -1;
    }
    // post-activation buffers: stem, conv1/conv2/conv3 of each block (downsample shares conv3's)
    t.conv[0].a = take((long long)B * 112 * 112 * 64);
    t.p0 = take((long long)B * 56 * 56 * 64);
    t.p0_idx = take(((long long)B * 56 * 56 * 64 + 3) / 4);
    for (const Block& b : n.blocks)
        for (int ci : {b.c1, b.c2, b.c3}) {
            const ConvLayer& c = n.convs[ci];
            t.conv[ci].a = take((long long)B * c.hout * c.hout * c.cout);
        }
    t.acc = take((long long)n.convs.size() * B * 16);
    t.xc = take(3LL * B * HEAD_LD);
    t.h1pre = take(3LL * B * HID); t.h1post = take(3LL * B * HID);
    t.h2pre = take(3LL * B * HID); t.h2post = take(3LL * B * HID);
    t.params = take(4LL * B * DEC_LD);
    t.masks = take(6LL * B * HID);
    t.total = off;
    return t;
}

static const Tape& tape_for(int B) {
    static std::vector<Tape> cache(65);
    static std::vector<char> ready(65, 0);
    if (!ready[B]) { cache[B] = build_tape(B); ready[B] = 1; }
    return cache[B];
}

static const long long kConvWs = 8LL << 20;    // split-K workspace (floats)

struct Scratch {
    float *ws, *g0, *g1, *t1, *t2, *t3, *t4, *t5, *t6, *gnp, *dP, *dy_dec, *d_h2, *d_h1, *dxc, *dxf, *tmp1024, *lin_ws;
    float *bsums, *bdgb;            // fused backward: fixed-point GroupNorm-backward sums [conv][B][4][2] and (d gamma, d beta) [channel][2] (long long)
    long long bacc_floats, gnp_floats;
    long long total;
    long long lin_ws_floats;
    Scratch(float* base, int B) {
        const long long S = (long long)B * 112 * 112 * 64;
        long long off = 0;
        auto take = [&](long long cnt) { float* p = base ? base + off : nullptr; off = align32(off + cnt); return p; };
        ws = take(kConvWs);
        g0 = take(S); g1 = take(S); t1 = take(S); t2 = take(S); t3 = take(S); t4 = take(S); t5 = take(S); t6 = take(S);
        long long gsum = 0;                               // per-sample dgamma / dbeta rows of EVERY GroupNorm (reduced once, at the end)
        for (const ConvLayer& c : net().convs) gsum += (long long)gn_bwd_partial_floats(B, c.hout * c.hout, c.cout);
        gnp = take(gsum);
        gnp_floats = gsum;
        long long csum = 0;
        for (const ConvLayer& c : net().convs) csum += c.cout;
        bsums = take((long long)net().convs.size() * B * 16);
        bdgb = take(csum * 4);
        bacc_floats = (long long)((bdgb + csum * 4) - bsums);
        dP = take((long long)B * DEC_LD);
        dy_dec = take(3LL * B * DEC_LD);
        d_h2 = take(3LL * B * HID); d_h1 = take(3LL * B * HID);
        dxc = take((long long)B * HEAD_LD);
        dxf = take((long long)B * 2048);
        tmp1024 = take((long long)B * HID);
        lin_ws_floats = 32LL * B * HEAD_LD;
        lin_ws = take(lin_ws_floats);
        total = off;
    }
};

// Weight gradients run on two library-owned side streams (alternating): every wgrad only needs (dy of its layer, the saved input
// activation) and writes its own slice of the gradient arena, so the chain  gn_bwd -> dgrad -> gn_bwd -> ...  on the
// caller's stream never waits for them.  At batch 1 each kernel fills a fraction of the SMs, and the two chains
// overlap.  Buffers read by a pending wgrad are protected by per-buffer events; the side stream is joined before return.
struct BwdAsync {
    static const int NSIDE = 2;
    cudaStream_t side[NSIDE] = {nullptr, nullptr};
    int next_side = 0;
    cudaEvent_t ev_ready[8];      // main -> side: "dy is ready" (ring)
    cudaEvent_t ev_read[8];       // side -> main: "buffer k has been read"
    cudaEvent_t ev_join[NSIDE];
    bool pending[8];
    int ring = 0;
    bool ok = false;
    bool init() {
        if (ok) return true;
        for (int i = 0; i < NSIDE; ++i)
            if (cudaStreamCreateWithFlags(&side[i], cudaStreamNonBlocking) != cudaSuccess) return false;
        for (int i = 0; i < 8; ++i) {
            if (cudaEventCreateWithFlags(&ev_ready[i], cudaEventDisableTiming) != cudaSuccess) return false;
            if (cudaEventCreateWithFlags(&ev_read[i], cudaEventDisableTiming) != cudaSuccess) return false;
            pending[i] = false;
        }
        for (int i = 0; i < NSIDE; ++i)
            if (cudaEventCreateWithFlags(&ev_join[i], cudaEventDisableTiming) != cudaSuccess) return false;
        ok = true;
        return true;
    }
};
static BwdAsync g_async;

// One process drives one GPU (one rank per GPU, as bench.py / torchrun launch it): the side streams and event rings above, the
// tensor-map caches and the per-function attribute cache of launch_ex belong to the device that was current at the first
// call.  A call from another device is refused (DBOA_ERR_UNSUPPORTED) instead of failing later with invalid-handle errors.
static int device_guard() {
    static int first = -1;
    int d = -1;
    if (cudaGetDevice(&d) != cudaSuccess) return DBOA_ERR_CUDA;
    if (first < 0) first = d;
    return d == first ? DBOA_OK : DBOA_ERR_UNSUPPORTED;
}

// Gradient buckets for the data-parallel all-reduce (SURVEY.md section 8e: "bucketed in reverse layer order and overlapped with
// backward").  The backward produces gradients head -> layer4 -> ... -> stem; the arena is laid out stem, layer1..4, head.
// Bucket 0 = [layer4 .. end), 1 = [layer3, layer4), 2 = [0, layer3).  When a caller hands over three events, event k is
// recorded once every kernel that writes bucket k (main chain, weight-gradient side streams, GroupNorm finish) has been
// enqueued and ordered before it; the caller's communication stream waits on it and all-reduces that span while the rest of
// the backward is still running.
struct BucketReq { cudaEvent_t ev[3]; bool armed; };
static BucketReq g_bucket_req = {{nullptr, nullptr, nullptr}, false};
static cudaStream_t g_join_stream = nullptr;
static cudaEvent_t g_join_ev[4] = {nullptr, nullptr, nullptr, nullptr};
void hmr_arm_bucket_events(cudaEvent_t e0, cudaEvent_t e1, cudaEvent_t e2) { g_bucket_req.ev[0] = e0; g_bucket_req.ev[1] = e1; g_bucket_req.ev[2] = e2; g_bucket_req.armed = true; }
long long hmr_bucket_offset(int k) {        // first float of bucket k's span; bucket k = [offset(k), offset(k - 1)) with offset(-1) = arena size
    const Net& n = net();
    if (k <= -1) return n.arena_floats;
    if (k >= 2) return 0;
    const char* first = k == 0 ? "layer4.0.conv1" : "layer3.0.conv1";
    for (const ConvLayer& c : n.convs)
        if (c.wname == first) return c.w_off;
    return 0;
}
// DBOA_ASYNC_WGRAD=0 in the environment keeps everything on the caller's stream (A/B measurements, debugging)
static const bool g_async_enabled = [] { const char* e = getenv("DBOA_ASYNC_WGRAD"); return !(e && e[0] == '0'); }();

static ConvDims dims_of(const ConvLayer& c, int B, int groups = 1, unsigned long long active = ~0ULL);

// Fused plan (conv_tc.cu with an operand transform): every convolution applies the GroupNorm (+ residual, ReLU) of its operand on
// load and leaves the statistics of its output as fixed-point sums; the fused data gradient applies GroupNorm backward on load
// and produces the sums of the next GroupNorm backward in its epilogue.  Both plans fill the same tape.  The default is one
// convolution and one GroupNorm launch per layer: on an H100 SXM (700 W) the fused plan measured 65.7 adapted frames/s for C2
// against 129.0, since the per-element transform in the loader costs more than the launches it saves.  DBOA_FUSED_FWD=1 / DBOA_FUSED_BWD=1 (or dboa_set_fused_forward(1) / dboa_set_fused_backward(1)) select it.
static bool g_fused_bwd = [] { const char* e = getenv("DBOA_FUSED_BWD"); return e && e[0] == '1'; }();
void hmr_set_fused_backward(bool on) { g_fused_bwd = on; }
static bool g_fused_fwd = [] { const char* e = getenv("DBOA_FUSED_FWD"); return e && e[0] == '1'; }();
void hmr_set_fused_forward(bool on) { g_fused_fwd = on; }
bool hmr_fused_forward() { return g_fused_fwd; }
bool hmr_fused_backward() { return g_fused_bwd; }

// table for gn_param_finish: where each GroupNorm's affine gradients live and where its per-sample rows start (the device copy
// is made by hmr_prepare)
struct GnItems { std::vector<long long> cum; std::vector<GnFinishItem> host; GnFinishItem* dev = nullptr; };
static GnItems& gn_items() {
    static GnItems gi = [] {
        GnItems g;
        long long cum = 0;
        for (const ConvLayer& c : net().convs) {
            g.cum.push_back(cum);
            g.host.push_back(GnFinishItem{c.g_off, c.b_off, cum, c.cout});
            cum += c.cout;
        }
        return g;
    }();
    return gi;
}

// Everything the backward creates once: the weight-gradient side streams and events, the data-parallel join stream and events,
// the GroupNorm item table on the device and the GroupNorm sync words.  Made by the first backward, or ahead of a CUDA graph
// capture by dboa_prepare_graph (while a stream captures, none of it may be created: the capture would be invalidated).
static bool g_prepared = false;
int hmr_prepare() {
    if (g_prepared) return DBOA_OK;
    DBOA_TRY(device_guard());
    if (!g_async.init()) return DBOA_ERR_CUDA;
    if (g_join_stream == nullptr && cudaStreamCreateWithFlags(&g_join_stream, cudaStreamNonBlocking) != cudaSuccess) return DBOA_ERR_CUDA;
    for (int i = 0; i < 4; ++i)
        if (g_join_ev[i] == nullptr && cudaEventCreateWithFlags(&g_join_ev[i], cudaEventDisableTiming) != cudaSuccess) return DBOA_ERR_CUDA;
    GnItems& gi = gn_items();
    if (gi.dev == nullptr) {
        void* p = nullptr;
        const size_t bytes = gi.host.size() * sizeof(GnFinishItem);
        if (cudaMalloc(&p, bytes) != cudaSuccess) return DBOA_ERR_CUDA;
        if (cudaMemcpy(p, gi.host.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(p); return DBOA_ERR_CUDA; }
        gi.dev = static_cast<GnFinishItem*>(p);
    }
    DBOA_TRY(gn_prepare());
    g_prepared = true;
    return DBOA_OK;
}

// backward convolutions: wgmma implicit GEMM when enabled and the shape is taken, else the fp32 CUDA-core kernels
static int conv_backward_data(const ConvLayer& c, int B, int groups, unsigned long long active, const float* dy, const float* w, float* dx,
                              int accumulate, float* ws, cudaStream_t st);
static int conv_backward_weight(const ConvLayer& c, int B, int groups, unsigned long long active, const float* dy, const float* x, float* dw,
                                float* ws, cudaStream_t st);

// B samples in `groups` videos of B / groups consecutive samples; video g's weights (and weight gradients) are one arena further on;
// the videos whose `active` bit is clear are skipped
static ConvDims dims_of(const ConvLayer& c, int B, int groups, unsigned long long active) {
    ConvDims d;
    d.B = B / groups; d.groups = groups; d.wstride = net().arena_floats; d.active = active;
    d.Hi = c.hin; d.Wi = c.hin; d.Cin = c.cin; d.Ho = c.hout; d.Wo = c.hout; d.Cout = c.cout;
    d.kh = c.k; d.kw = c.k; d.stride = c.stride; d.pad = c.pad; d.Kpitch = c.kpitch;
    return d;
}

// conv forward: wgmma implicit GEMM when enabled and the shape is taken (Cin % 64 == 0, Cout % 64 == 0), else the fp32 CUDA-core kernel
static int conv_forward(const ConvLayer& c, int B, int groups, unsigned long long active, const float* x, const float* w, float* y, float* ws,
                        cudaStream_t st) {
    const ConvDims d = dims_of(c, B, groups, active);
    if (conv_tc_enabled()) {
        int s = conv_tc_fwd(x, w, y, d, st);
        if (s != DBOA_ERR_UNSUPPORTED) return s;
    }
    return conv_fwd(x, w, y, d, ws, (size_t)kConvWs, st);
}

static int conv_backward_data(const ConvLayer& c, int B, int groups, unsigned long long active, const float* dy, const float* w, float* dx,
                              int accumulate, float* ws, cudaStream_t st) {
    const ConvDims d = dims_of(c, B, groups, active);
    if (conv_tc_bwd_enabled()) {
        int s = conv_tc_dgrad(dy, w, dx, d, accumulate, st);
        if (s != DBOA_ERR_UNSUPPORTED) return s;
    }
    return conv_dgrad(dy, w, dx, d, accumulate, ws, (size_t)kConvWs, st);
}
static int conv_backward_weight(const ConvLayer& c, int B, int groups, unsigned long long active, const float* dy, const float* x, float* dw,
                                float* ws, cudaStream_t st) {
    const ConvDims d = dims_of(c, B, groups, active);
    if (conv_tc_wgrad_enabled()) {
        int s = conv_tc_wgrad(dy, x, dw, d, st);
        if (s != DBOA_ERR_UNSUPPORTED) return s;
    }
    return conv_wgrad(dy, x, dw, d, ws, (size_t)kConvWs, st);
}

// Argument checks of a grouped call (host only, before any device access).  Video g owns samples [g * B / groups, (g + 1) * B /
// groups) and the arena, gradient arena and weights one arena_floats apart; only the default plan serves several videos, and the
// data-parallel gradient buckets (one arena, all-reduced across ranks) do not apply to them.  `active` (bit g: video g takes part)
// must name at least one video and none past `groups`.
static int groups_check(int B, int groups, unsigned long long active) {
    if (groups < 1 || B < 1 || B > 64 || B % groups != 0) return DBOA_ERR_SHAPE;
    if (active == 0 || (groups < 64 && (active >> groups) != 0)) return DBOA_ERR_ARG;
    if (groups > 1 && (g_fused_fwd || g_fused_bwd)) return DBOA_ERR_UNSUPPORTED;
    return DBOA_OK;
}

__global__ void head_init_kernel(const float* __restrict__ ip, const float* __restrict__ is, const float* __restrict__ ic,
                                 float* __restrict__ params0, float* __restrict__ xc0, int B) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * NDEC) return;
    int b = i / NDEC, j = i - b * NDEC;
    float v = j < 144 ? ip[j] : (j < 154 ? is[j - 144] : ic[j - 154]);
    params0[(size_t)b * DEC_LD + j] = v;
    xc0[(size_t)b * HEAD_LD + 2048 + j] = v;
}
__global__ void head_out_kernel(const float* __restrict__ params3, float* __restrict__ shape, float* __restrict__ cam,
                                float* __restrict__ pose6d, int B) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * NDEC) return;
    int b = i / NDEC, j = i - b * NDEC;
    float v = params3[(size_t)b * DEC_LD + j];
    if (j < 144) { if (pose6d) pose6d[(size_t)b * 144 + j] = v; }
    else if (j < 154) shape[(size_t)b * 10 + (j - 144)] = v;
    else cam[(size_t)b * 3 + (j - 154)] = v;
}
// dP[b][:] = [rot6d-adjoint (filled separately) | d_shape | d_cam]
__global__ void head_grad_in_kernel(const float* __restrict__ dshape, const float* __restrict__ dcam, float* __restrict__ dP, int B) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 16) return;
    int b = i / 16, j = i - b * 16;
    float v = j < 10 ? (dshape ? dshape[b * 10 + j] : 0.f) : (j < 13 ? (dcam ? dcam[b * 3 + (j - 10)] : 0.f) : 0.f);
    dP[(size_t)b * DEC_LD + 144 + j] = v;
}
// pose6d rows live with a leading dimension (DEC_LD) inside the tape
__global__ void rot6d_rows_fwd_kernel(const float* __restrict__ params3, float* __restrict__ rotmat, int B);
__global__ void rot6d_rows_bwd_kernel(const float* __restrict__ params3, const float* __restrict__ drot, float* __restrict__ dP, int B);

}  // namespace dboa

#include "rotmath.cuh"
namespace dboa {

__global__ void rot6d_rows_fwd_kernel(const float* __restrict__ params3, float* __restrict__ rotmat, int B) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 24) return;
    int b = i / 24, j = i - b * 24;
    float x[6], R[9];
    for (int k = 0; k < 6; ++k) x[k] = params3[(size_t)b * DEC_LD + j * 6 + k];
    rot6d_fwd(x, R);
    for (int k = 0; k < 9; ++k) rotmat[(size_t)i * 9 + k] = R[k];
}
__global__ void rot6d_rows_bwd_kernel(const float* __restrict__ params3, const float* __restrict__ drot, float* __restrict__ dP, int B) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 24) return;
    int b = i / 24, j = i - b * 24;
    float x[6], g[9], d[6];
    for (int k = 0; k < 6; ++k) x[k] = params3[(size_t)b * DEC_LD + j * 6 + k];
    for (int k = 0; k < 9; ++k) g[k] = drot ? drot[(size_t)i * 9 + k] : 0.f;
    rot6d_bwd(x, g, d);
    for (int k = 0; k < 6; ++k) dP[(size_t)b * DEC_LD + j * 6 + k] = d[k];
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
int hmr_forward(const float* P, const float* init_pose, const float* init_shape, const float* init_cam, const float* image, int B,
                const float* drop_masks, float* T, float* scratch, float* rotmat, float* shape, float* cam, float* pose6d,
                cudaStream_t st, int groups, unsigned long long active) {
    DBOA_TRY(groups_check(B, groups, active));
    DBOA_TRY(device_guard());
    const Net& n = net();
    const long long PS = n.arena_floats;
    const Tape& t = tape_for(B);
    Scratch sc(scratch, B);
    auto gn_plain = [&](int ci, float* out, int relu, const float* res) {
        const ConvLayer& c = n.convs[ci];
        int HW = c.hout * c.hout;
        return gn_fwd_fused(T + t.conv[ci].y, P + c.g_off, P + c.b_off, res, out, T + t.conv[ci].stats, T + t.conv[ci].part, B, HW,
                            c.cout, relu, st, B / groups, PS);
    };
    if (g_fused_fwd && conv_tc_enabled())
        cudaMemsetAsync(T + t.acc, 0, n.convs.size() * (size_t)B * 16 * sizeof(float), st);      // statistics accumulators of this forward
    DBOA_TRY(nchw_to_nhwc(image, T + t.x0, B, 3, 224, 224, st));
    DBOA_TRY(conv_forward(n.convs[0], B, groups, active, T + t.x0, P + n.convs[0].w_off, T + t.conv[0].y, sc.ws, st));
    DBOA_TRY(gn_plain(0, T + t.conv[0].a, 1, nullptr));
    DBOA_TRY(maxpool3x3s2_fwd(T + t.conv[0].a, T + t.p0, reinterpret_cast<unsigned char*>(T + t.p0_idx), B, 112, 112, 64, st));
    const float* x = T + t.p0;
    if (g_fused_fwd && conv_tc_enabled()) {
        // ---- fused plan (conv_tc.cu operand transform): every convolution applies the GroupNorm (+ residual, ReLU) of its operand on
        // load and leaves the statistics of its output as fixed-point sums; one launch per convolution.
        auto acc_of = [&](int ci) { return T + t.acc + (long long)ci * B * 16; };
        auto base_desc = [&](int ci) {
            const ConvLayer& c = n.convs[ci];
            FusedConv f;
            memset(&f, 0, sizeof f);
            f.w = P + c.w_off; f.y = T + t.conv[ci].y; f.part_out = acc_of(ci);
            f.Hi = c.hin; f.Cin = c.cin; f.Cout = c.cout; f.k = c.k; f.stride = c.stride; f.pad = c.pad; f.Ho = c.hout;
            return f;
        };
        auto gn_of = [&](FusedConv& f, int src) {                  // operand = relu(gn(y[src])), materialised into the tape on the way
            const ConvLayer& c = n.convs[src];
            f.mode = 1; f.x = T + t.conv[src].y; f.part_in = acc_of(src);
            f.gamma = P + c.g_off; f.beta = P + c.b_off;
            f.a_out = T + t.conv[src].a; f.stats_out = T + t.conv[src].stats;
        };
        auto run = [&](FusedConv* d, int np) { return conv_fused_fwd(d, np, B, st, true); };
        for (size_t bi = 0; bi < n.blocks.size(); ++bi) {
            const Block& b = n.blocks[bi];
            // ---- conv1 (+ the shortcut convolution in the same launch: both read the previous block's output, formed on load)
            FusedConv d[2];
            const int np = b.cd >= 0 ? 2 : 1;
            const int ci[2] = {b.c1, b.cd};
            for (int i = 0; i < np; ++i) {
                FusedConv& f = d[i];
                f = base_desc(ci[i]);
                if (bi == 0) { f.mode = 0; f.x = T + t.p0; continue; }
                const Block& pb = n.blocks[bi - 1];
                gn_of(f, pb.c3);
                if (pb.cd >= 0) {
                    const ConvLayer& pd = n.convs[pb.cd];
                    f.mode = 3; f.res = T + t.conv[pb.cd].y; f.part2_in = acc_of(pb.cd);
                    f.gamma2 = P + pd.g_off; f.beta2 = P + pd.b_off; f.stats2_out = T + t.conv[pb.cd].stats;
                } else {
                    f.mode = 2; f.res = bi >= 2 ? T + t.conv[n.blocks[bi - 2].c3].a : T + t.p0;
                }
                if (i == 1) { f.a_out = nullptr; f.stats_out = nullptr; f.stats2_out = nullptr; }     // conv1 is the writer
            }
            DBOA_TRY(run(d, np));
            d[0] = base_desc(b.c2); gn_of(d[0], b.c1);
            DBOA_TRY(run(d, 1));
            d[0] = base_desc(b.c3); gn_of(d[0], b.c2);
            DBOA_TRY(run(d, 1));
        }
        const Block& lb = n.blocks.back();
        const ConvLayer& l3 = n.convs[lb.c3];
        if (lb.cd >= 0) return DBOA_ERR_UNSUPPORTED;
        DBOA_TRY(gn_acc_res_avgpool(T + t.conv[lb.c3].y, T + t.conv[n.blocks[n.blocks.size() - 2].c3].a, acc_of(lb.c3), P + l3.g_off, P + l3.b_off,
                                    T + t.conv[lb.c3].a, T + t.conv[lb.c3].stats, T + t.xc, B, 49, 2048, HEAD_LD, 3, (size_t)B * HEAD_LD, st));
    } else {
    for (const Block& b : n.blocks) {
        const ConvLayer &c1 = n.convs[b.c1], &c2 = n.convs[b.c2], &c3 = n.convs[b.c3];
        DBOA_TRY(conv_forward(c1, B, groups, active, x, P + c1.w_off, T + t.conv[b.c1].y, sc.ws, st));
        DBOA_TRY(gn_plain(b.c1, T + t.conv[b.c1].a, 1, nullptr));
        DBOA_TRY(conv_forward(c2, B, groups, active, T + t.conv[b.c1].a, P + c2.w_off, T + t.conv[b.c2].y, sc.ws, st));
        DBOA_TRY(gn_plain(b.c2, T + t.conv[b.c2].a, 1, nullptr));
        DBOA_TRY(conv_forward(c3, B, groups, active, T + t.conv[b.c2].a, P + c3.w_off, T + t.conv[b.c3].y, sc.ws, st));
        const int HW = c3.hout * c3.hout;
        if (b.cd >= 0) {
            const ConvLayer& cd = n.convs[b.cd];
            DBOA_TRY(conv_forward(cd, B, groups, active, x, P + cd.w_off, T + t.conv[b.cd].y, sc.ws, st));
            (void)HW;
            DBOA_TRY(gn_plain(b.cd, sc.t1, 0, nullptr));                 // normalised shortcut -> scratch
            DBOA_TRY(gn_plain(b.c3, T + t.conv[b.c3].a, 1, sc.t1));      // relu(gn(y3) + shortcut)
        } else {
            DBOA_TRY(gn_plain(b.c3, T + t.conv[b.c3].a, 1, x));
        }
        x = T + t.conv[b.c3].a;
    }
    // pooled feature goes straight into the three regressor input rows
    DBOA_TRY(avgpool_fwd(x, T + t.xc, B, 49, 2048, HEAD_LD, 3, (size_t)B * HEAD_LD, st));
    }
    DBOA_TRY(launch_ex(head_init_kernel, dim3(ceil_div(B * NDEC, 128)), dim3(128), 0, st, dim3(1, 1, 1), true, init_pose, init_shape, init_cam, T + t.params, T + t.xc, B));
    if (drop_masks) cudaMemcpyAsync(T + t.masks, drop_masks, 6ULL * B * HID * sizeof(float), cudaMemcpyDeviceToDevice, st);
    for (int it = 0; it < 3; ++it) {
        const float* m1 = drop_masks ? T + t.masks + (size_t)(it * 2 + 0) * B * HID : nullptr;
        const float* m2 = drop_masks ? T + t.masks + (size_t)(it * 2 + 1) * B * HID : nullptr;
        float* xc = T + t.xc + (size_t)it * B * HEAD_LD;
        float* h1pre = T + t.h1pre + (size_t)it * B * HID; float* h1post = T + t.h1post + (size_t)it * B * HID;
        float* h2pre = T + t.h2pre + (size_t)it * B * HID; float* h2post = T + t.h2post + (size_t)it * B * HID;
        DBOA_TRY(linear_fwd(xc, HEAD_LD, P + n.fc1_w, HEAD_LD, P + n.fc1_b, nullptr, 0, m1, h1pre, h1post, HID, nullptr, 0, B, HID, HEAD_IN, st,
                            groups, PS, active));
        DBOA_TRY(linear_fwd(h1post, HID, P + n.fc2_w, HID, P + n.fc2_b, nullptr, 0, m2, h2pre, h2post, HID, nullptr, 0, B, HID, HID, st, groups, PS, active));
        float* pin = T + t.params + (size_t)it * B * DEC_LD;
        float* pout = T + t.params + (size_t)(it + 1) * B * DEC_LD;
        float* xnext = it < 2 ? T + t.xc + (size_t)(it + 1) * B * HEAD_LD + 2048 : nullptr;
        DBOA_TRY(linear_fwd(h2post, HID, P + n.dec_w, HID, P + n.dec_b, pin, DEC_LD, nullptr, nullptr, pout, DEC_LD, xnext, HEAD_LD, B, NDEC,
                            HID, st, groups, PS, active));
    }
    const float* p3 = T + t.params + 3ULL * B * DEC_LD;
    DBOA_TRY(launch_ex(rot6d_rows_fwd_kernel, dim3(ceil_div(B * 24, 128)), dim3(128), 0, st, dim3(1, 1, 1), true, p3, rotmat, B));
    return launch_ex(head_out_kernel, dim3(ceil_div(B * NDEC, 128)), dim3(128), 0, st, dim3(1, 1, 1), true, p3, shape, cam, pose6d, B);
}

// ---------------------------------------------------------------------------------------------
// backward (accumulates into the flat gradient arena G, same layout as P)
// ---------------------------------------------------------------------------------------------
int hmr_backward(const float* P, const float* T, int B, int masked_in, const float* d_rotmat, const float* d_shape, const float* d_cam,
                 float* G, float* scratch, cudaStream_t st, int groups, unsigned long long active) {
    const bool bucketed = g_bucket_req.armed;
    if (groups != 1) g_bucket_req.armed = false;         // a request armed for a grouped call is consumed by it, whatever it returns
    DBOA_TRY(groups_check(B, groups, active));
    if (groups > 1 && bucketed) return DBOA_ERR_UNSUPPORTED;
    DBOA_TRY(device_guard());
    const Net& n = net();
    const long long PS = n.arena_floats;
    const Tape& t = tape_for(B);
    Scratch sc(scratch, B);
    const bool masked = masked_in != 0;     // the forward ran with dropout keep-masks (saved in the tape)
    BucketReq breq = g_bucket_req;
    g_bucket_req.armed = false;
    if (!g_prepared) {
        if (stream_capturing(st)) return DBOA_ERR_UNSUPPORTED;
        DBOA_TRY(hmr_prepare());
    }

    // ---- head
    const float* p3 = T + t.params + 3ULL * B * DEC_LD;
    cudaMemsetAsync(sc.dP, 0, (size_t)B * DEC_LD * sizeof(float), st);
    DBOA_TRY(launch_ex(rot6d_rows_bwd_kernel, dim3(ceil_div(B * 24, 128)), dim3(128), 0, st, dim3(1, 1, 1), true, p3, d_rotmat, sc.dP, B));
    DBOA_TRY(launch_ex(head_grad_in_kernel, dim3(ceil_div(B * 16, 128)), dim3(128), 0, st, dim3(1, 1, 1), true, d_shape, d_cam, sc.dP, B));
    cudaMemsetAsync(sc.dxf, 0, (size_t)B * 2048 * sizeof(float), st);
    for (int it = 2; it >= 0; --it) {
        float* dy_dec = sc.dy_dec + (size_t)it * B * DEC_LD;
        float* d_h2 = sc.d_h2 + (size_t)it * B * HID;
        float* d_h1 = sc.d_h1 + (size_t)it * B * HID;
        cudaMemcpyAsync(dy_dec, sc.dP, (size_t)B * DEC_LD * sizeof(float), cudaMemcpyDeviceToDevice, st);
        if (masked) {
            DBOA_TRY(linear_dgrad(dy_dec, DEC_LD, P + n.dec_w, HID, sc.tmp1024, HID, B, NDEC, HID, sc.lin_ws, sc.lin_ws_floats, st, groups, PS, active));
            DBOA_TRY(ew_mul(sc.tmp1024, T + t.masks + (size_t)(it * 2 + 1) * B * HID, d_h2, (size_t)B * HID, st));
            DBOA_TRY(linear_dgrad(d_h2, HID, P + n.fc2_w, HID, sc.tmp1024, HID, B, HID, HID, sc.lin_ws, sc.lin_ws_floats, st, groups, PS, active));
            DBOA_TRY(ew_mul(sc.tmp1024, T + t.masks + (size_t)(it * 2 + 0) * B * HID, d_h1, (size_t)B * HID, st));
        } else {
            DBOA_TRY(linear_dgrad(dy_dec, DEC_LD, P + n.dec_w, HID, d_h2, HID, B, NDEC, HID, sc.lin_ws, sc.lin_ws_floats, st, groups, PS, active));
            DBOA_TRY(linear_dgrad(d_h2, HID, P + n.fc2_w, HID, d_h1, HID, B, HID, HID, sc.lin_ws, sc.lin_ws_floats, st, groups, PS, active));
        }
        DBOA_TRY(linear_dgrad(d_h1, HID, P + n.fc1_w, HEAD_LD, sc.dxc, HEAD_LD, B, HID, HEAD_IN, sc.lin_ws, sc.lin_ws_floats, st, groups, PS, active));
        DBOA_TRY(ew_add_rows(sc.dxf, 2048, sc.dxf, 2048, sc.dxc, HEAD_LD, B, 2048, st));
        DBOA_TRY(ew_add_rows(sc.dP, DEC_LD, sc.dP, DEC_LD, sc.dxc + 2048, HEAD_LD, B, NDEC, st));
    }
    DBOA_TRY(linear_wgrad(sc.dy_dec, DEC_LD, T + t.h2post, HID, G + n.dec_w, HID, G + n.dec_b, 3 * B, NDEC, HID, st, groups, B, PS, active));
    DBOA_TRY(linear_wgrad(sc.d_h2, HID, T + t.h1post, HID, G + n.fc2_w, HID, G + n.fc2_b, 3 * B, HID, HID, st, groups, B, PS, active));
    DBOA_TRY(linear_wgrad(sc.d_h1, HID, T + t.xc, HEAD_LD, G + n.fc1_w, HEAD_LD, G + n.fc1_b, 3 * B, HID, HEAD_IN, st, groups, B, PS, active));

    // ---- backbone
    float* dOut = sc.g0;
    float* dIn = sc.g1;
    DBOA_TRY(avgpool_bwd(sc.dxf, 2048, dOut, B, 49, 2048, st));
    float* const tmp[6] = {sc.t1, sc.t2, sc.t3, sc.t4, sc.t5, sc.t6};
    const bool async = g_async_enabled;
    BwdAsync& A = g_async;
    if (async) {                                   // the side stream starts after everything enqueued so far
        for (int i = 0; i < 8; ++i) A.pending[i] = false;
        cudaEventRecord(A.ev_ready[A.ring], st);
        for (int i = 0; i < BwdAsync::NSIDE; ++i) cudaStreamWaitEvent(A.side[i], A.ev_ready[A.ring], 0);
        A.ring = (A.ring + 1) & 7;
    }
    // before the main chain overwrites temp k: wait for the weight-gradient kernel that still reads it
    auto claim = [&](int k) {
        if (async && A.pending[k]) { cudaStreamWaitEvent(st, A.ev_read[k], 0); A.pending[k] = false; }
        return tmp[k];
    };
    auto gnb = [&](int ci, const float* dout, const float* mask_src, float* dy) {
        const ConvLayer& c = n.convs[ci];
        return gn_bwd_fused(dout, mask_src, T + t.conv[ci].y, T + t.conv[ci].stats, P + c.g_off, dy, G + c.g_off, G + c.b_off,
                            sc.gnp + 2 * (size_t)B * gn_items().cum[ci], B, c.hout * c.hout, c.cout, st, /*defer=*/1, B / groups, PS);
    };
    // weight gradient of conv `c` from dy held in temp k
    auto wgrad = [&](const ConvLayer& c, int k, const float* xin_) {
        if (!async) return conv_backward_weight(c, B, groups, active, tmp[k], xin_, G + c.w_off, sc.ws, st);
        cudaStream_t ss = A.side[A.next_side];
        A.next_side = (A.next_side + 1) % BwdAsync::NSIDE;
        cudaEventRecord(A.ev_ready[A.ring], st);
        cudaStreamWaitEvent(ss, A.ev_ready[A.ring], 0);
        A.ring = (A.ring + 1) & 7;
        int s_ = conv_backward_weight(c, B, groups, active, tmp[k], xin_, G + c.w_off, sc.ws, ss);
        cudaEventRecord(A.ev_read[k], ss);
        A.pending[k] = true;
        return s_;
    };
    // gradients of convs [first_conv, ...) are complete (B > 1: their GroupNorm affine rows get summed here, not at the very end)
    int finished_from = (int)n.convs.size();
    auto bucket_done = [&](int k, int first_conv) {
        if (B > 1 && first_conv < finished_from) {
            const GnItems& gi = gn_items();
            DBOA_TRY(gn_param_finish(gi.dev + first_conv, finished_from - first_conv, sc.gnp, G, B, st, groups, PS, active));
            finished_from = first_conv;
        }
        if (!breq.armed) return DBOA_OK;
        cudaEventRecord(g_join_ev[0], st);
        cudaStreamWaitEvent(g_join_stream, g_join_ev[0], 0);
        if (async)
            for (int i = 0; i < BwdAsync::NSIDE; ++i) {
                cudaEventRecord(g_join_ev[1 + i], A.side[i]);
                cudaStreamWaitEvent(g_join_stream, g_join_ev[1 + i], 0);
            }
        cudaEventRecord(breq.ev[k], g_join_stream);
        return DBOA_OK;
    };
    const bool fused = g_fused_bwd && conv_tc_bwd_enabled();
    if (fused) {
        // ---- fused chain (conv_tc.cu, GroupNorm backward on load): per stride-1 layer ONE launch does GroupNorm backward (on load), the data gradient, the
        // shortcut add, the ReLU mask of the producing layer and the sums of ITS GroupNorm backward; the stride-2 layers (conv2
        // and shortcut of layer2.0 / 3.0 / 4.0) keep the unfused kernels, stitched in with gn_bwd_prep.
        auto sums_of = [&](int ci) { return sc.bsums + (long long)ci * B * 16; };
        auto dgb_of = [&](int ci) { return sc.bdgb + 4 * gn_items().cum[ci]; };
        auto prep_of = [&](int ci) {
            const ConvLayer& c = n.convs[ci];
            DgradPrep p;
            p.y = T + t.conv[ci].y; p.stats = T + t.conv[ci].stats; p.gamma = P + c.g_off; p.sums = sums_of(ci); p.dgb = dgb_of(ci);
            return p;
        };
        auto K = [&](int ci, const float* dzin, float* dy_out, const float* addend, float* out, const float* mask, int np, int p0, int p1) {
            const ConvLayer& c = n.convs[ci];
            DgradFused f;
            memset(&f, 0, sizeof f);
            f.dz = dzin; f.y_c = T + t.conv[ci].y; f.w = P + c.w_off; f.stats_c = T + t.conv[ci].stats; f.sums_c = sums_of(ci); f.gamma_c = P + c.g_off;
            f.dy_out = dy_out; f.addend = addend; f.out = out; f.mask = mask; f.nprep = mask ? np : 0;
            if (mask && np >= 1) f.prep[0] = prep_of(p0);
            if (mask && np >= 2) f.prep[1] = prep_of(p1);
            return dgrad_fused(f, dims_of(c, B), st, true);
        };
        cudaMemsetAsync(sc.bsums, 0, (size_t)sc.bacc_floats * sizeof(float), st);
        if (B > 1) cudaMemsetAsync(sc.gnp, 0, (size_t)sc.gnp_floats * sizeof(float), st);       // rows of the layers that stay fused are never written
        {   // seam: dA of the last block's output -> masked gradient + sums of its bn3
            const Block& lb = n.blocks.back();
            DBOA_TRY(gn_bwd_prep(dOut, T + t.conv[lb.c3].a, dOut, prep_of(lb.c3), B, 49, 2048, st));
        }
        auto finish_fixed = [&](int first_conv, int end_conv) {
            const GnItems& gi = gn_items();
            return gn_dgb_finish(gi.dev + first_conv, end_conv - first_conv, sc.bdgb, G, st);
        };
        int fixed_from = (int)n.convs.size();
        for (int bi = (int)n.blocks.size() - 1; bi >= 0; --bi) {
            const Block& b = n.blocks[bi];
            const ConvLayer &c1 = n.convs[b.c1], &c2 = n.convs[b.c2], &c3 = n.convs[b.c3];
            if (bi == 12 || bi == 6) {
                const int first = bi == 12 ? n.blocks[13].c1 : n.blocks[7].c1;
                DBOA_TRY(finish_fixed(first, fixed_from));
                fixed_from = first;
                DBOA_TRY(bucket_done(bi == 12 ? 0 : 1, first));
            }
            const float* xin = bi == 0 ? T + t.p0 : T + t.conv[n.blocks[bi - 1].c3].a;
            const float* a3 = T + t.conv[b.c3].a;
            float* dzo = dOut;                                  // masked gradient w.r.t. this block's pre-ReLU output (sums of bn3 [and the fused shortcut's norm] filled)
            const bool sblock = c2.stride != 1;
            if (!sblock) {
                DBOA_TRY(K(b.c3, dzo, claim(0), nullptr, tmp[2], T + t.conv[b.c2].a, 1, b.c2, -1));
                DBOA_TRY(wgrad(c3, 0, T + t.conv[b.c2].a));
                DBOA_TRY(K(b.c2, tmp[2], claim(3), nullptr, tmp[4], T + t.conv[b.c1].a, 1, b.c1, -1));
                DBOA_TRY(wgrad(c2, 3, T + t.conv[b.c1].a));
                const float* addend = dzo;                      // identity shortcut: d(out) flows straight to the block input
                if (b.cd >= 0) {                                // stride-1 shortcut convolution (layer1.0): its data gradient is the addend
                    DBOA_TRY(K(b.cd, dzo, claim(1), nullptr, dIn, nullptr, 0, -1, -1));
                    DBOA_TRY(wgrad(n.convs[b.cd], 1, xin));
                    addend = dIn;
                }
                if (bi > 0) {
                    const Block& pb = n.blocks[bi - 1];
                    const bool two = pb.cd >= 0 && n.convs[pb.cd].stride == 1;
                    DBOA_TRY(K(b.c1, tmp[4], claim(5), addend, dIn, T + t.conv[pb.c3].a, two ? 2 : 1, pb.c3, pb.cd));
                } else {
                    DBOA_TRY(K(b.c1, tmp[4], claim(5), addend, dIn, nullptr, 0, -1, -1));
                }
                DBOA_TRY(wgrad(c1, 5, xin));
            } else {
                DBOA_TRY(K(b.c3, dzo, claim(0), nullptr, claim(2), nullptr, 0, -1, -1));     // plain dA2: conv2's GroupNorm backward stays unfused
                DBOA_TRY(wgrad(c3, 0, T + t.conv[b.c2].a));
                const ConvLayer& cd = n.convs[b.cd];
                DBOA_TRY(gnb(b.cd, dzo, a3, claim(1)));
                DBOA_TRY(wgrad(cd, 1, xin));
                DBOA_TRY(conv_backward_data(cd, B, groups, active, tmp[1], P + cd.w_off, dIn, 0, sc.ws, st));
                DBOA_TRY(gnb(b.c2, tmp[2], T + t.conv[b.c2].a, claim(3)));
                DBOA_TRY(wgrad(c2, 3, T + t.conv[b.c1].a));
                DBOA_TRY(conv_backward_data(c2, B, groups, active, tmp[3], P + c2.w_off, claim(4), 0, sc.ws, st));
                DBOA_TRY(gnb(b.c1, tmp[4], T + t.conv[b.c1].a, claim(5)));
                DBOA_TRY(wgrad(c1, 5, xin));
                DBOA_TRY(conv_backward_data(c1, B, groups, active, tmp[5], P + c1.w_off, dIn, 1, sc.ws, st));
                const Block& pb = n.blocks[bi - 1];             // seam: the previous block (last of its layer) has an identity shortcut
                const ConvLayer& p3 = n.convs[pb.c3];
                DBOA_TRY(gn_bwd_prep(dIn, T + t.conv[pb.c3].a, dIn, prep_of(pb.c3), B, p3.hout * p3.hout, p3.cout, st));
            }
            float* sw = dOut; dOut = dIn; dIn = sw;
        }
        DBOA_TRY(finish_fixed(0, fixed_from));
    } else {
    for (int bi = (int)n.blocks.size() - 1; bi >= 0; --bi) {
        const Block& b = n.blocks[bi];
        const ConvLayer &c1 = n.convs[b.c1], &c2 = n.convs[b.c2], &c3 = n.convs[b.c3];
        if (bi == 12) DBOA_TRY(bucket_done(0, n.blocks[13].c1));          // layer4 (blocks 13..15) and the head are done
        if (bi == 6) DBOA_TRY(bucket_done(1, n.blocks[7].c1));            // layer3 (blocks 7..12)
        const float* xin = bi == 0 ? T + t.p0 : T + t.conv[n.blocks[bi - 1].c3].a;
        const float* a3 = T + t.conv[b.c3].a;
        // temps: 0 = dy3, 1 = dy_downsample, 2 = da2, 3 = dy2, 4 = da1, 5 = dy1
        DBOA_TRY(gnb(b.c3, dOut, a3, claim(0)));
        DBOA_TRY(wgrad(c3, 0, T + t.conv[b.c2].a));
        if (b.cd >= 0) {
            const ConvLayer& cd = n.convs[b.cd];
            DBOA_TRY(gnb(b.cd, dOut, a3, claim(1)));
            DBOA_TRY(wgrad(cd, 1, xin));
            DBOA_TRY(conv_backward_data(cd, B, groups, active, tmp[1], P + cd.w_off, dIn, 0, sc.ws, st));
        } else {
            DBOA_TRY(relu_mask(dOut, a3, dIn, (size_t)B * c3.hout * c3.hout * c3.cout, st));
        }
        DBOA_TRY(conv_backward_data(c3, B, groups, active, tmp[0], P + c3.w_off, claim(2), 0, sc.ws, st));
        DBOA_TRY(gnb(b.c2, tmp[2], T + t.conv[b.c2].a, claim(3)));
        DBOA_TRY(wgrad(c2, 3, T + t.conv[b.c1].a));
        DBOA_TRY(conv_backward_data(c2, B, groups, active, tmp[3], P + c2.w_off, claim(4), 0, sc.ws, st));
        DBOA_TRY(gnb(b.c1, tmp[4], T + t.conv[b.c1].a, claim(5)));
        DBOA_TRY(wgrad(c1, 5, xin));
        DBOA_TRY(conv_backward_data(c1, B, groups, active, tmp[5], P + c1.w_off, dIn, 1, sc.ws, st));
        float* sw = dOut; dOut = dIn; dIn = sw;
    }
    }
    // ---- stem: maxpool, GroupNorm+ReLU, conv (weight gradient only; the image needs none)
    DBOA_TRY(maxpool3x3s2_bwd(dOut, reinterpret_cast<const unsigned char*>(T + t.p0_idx), dIn, B, 112, 112, 64, st));
    DBOA_TRY(gnb(0, dIn, T + t.conv[0].a, claim(0)));
    int rc = conv_wgrad(tmp[0], T + t.x0, G + n.convs[0].w_off, dims_of(n.convs[0], B, groups, active), sc.ws, (size_t)kConvWs, st);
    if (rc == DBOA_OK) rc = bucket_done(2, 0);               // stem, layer1, layer2 (and, for B > 1, their GroupNorm affine rows)
    if (async) {                                   // join: nothing of this call is left running when the caller's stream continues
        for (int i = 0; i < BwdAsync::NSIDE; ++i) {
            cudaEventRecord(A.ev_join[i], A.side[i]);
            cudaStreamWaitEvent(st, A.ev_join[i], 0);
        }
        for (int i = 0; i < 8; ++i) A.pending[i] = false;
    }
    return rc;
}

// ---------------------------------------------------------------------------------------------
// layout queries
// ---------------------------------------------------------------------------------------------
int hmr_num_params() { return (int)net().params.size(); }
long long hmr_arena_floats() { return net().arena_floats; }
int hmr_param_info(int i, char* name, int cap, long long* off, int* ndim, long long shape[4], long long stride[4]) {
    const Net& n = net();
    if (i < 0 || i >= (int)n.params.size()) return DBOA_ERR_ARG;
    const ParamInfo& p = n.params[i];
    if (name && cap > 0) { strncpy(name, p.name.c_str(), cap - 1); name[cap - 1] = 0; }
    *off = p.off; *ndim = p.ndim;
    for (int k = 0; k < 4; ++k) { shape[k] = p.shape[k]; stride[k] = p.stride[k]; }
    return DBOA_OK;
}
long long hmr_tape_floats(int B) { return (B < 1 || B > 64) ? -1 : tape_for(B).total; }
long long hmr_tape_offset(int B, int kind, int conv) {
    if (B < 1 || B > 64) return DBOA_ERR_SHAPE;
    const Tape& t = tape_for(B);
    if (kind == DBOA_TAPE_Y || kind == DBOA_TAPE_STATS || kind == DBOA_TAPE_A) {
        if (conv < 0 || conv >= (int)t.conv.size()) return DBOA_ERR_ARG;
        const ConvTape& c = t.conv[conv];
        if (kind == DBOA_TAPE_A && c.a < 0) return DBOA_ERR_ARG;         // downsample: the block's output is conv3's `a`
        return kind == DBOA_TAPE_Y ? c.y : (kind == DBOA_TAPE_STATS ? c.stats : c.a);
    }
    switch (kind) {
        case DBOA_TAPE_X0: return t.x0;
        case DBOA_TAPE_P0: return t.p0;
        case DBOA_TAPE_P0_IDX: return t.p0_idx;
        case DBOA_TAPE_XC: return t.xc;
        case DBOA_TAPE_H1PRE: return t.h1pre;
        case DBOA_TAPE_H1POST: return t.h1post;
        case DBOA_TAPE_H2PRE: return t.h2pre;
        case DBOA_TAPE_H2POST: return t.h2post;
        case DBOA_TAPE_PARAMS: return t.params;
        case DBOA_TAPE_MASKS: return t.masks;
        default: return DBOA_ERR_ARG;
    }
}
long long hmr_scratch_floats(int B) { return (B < 1 || B > 64) ? -1 : Scratch(nullptr, B).total; }
int hmr_feature_info(int B, int i, long long* off, int* ndim, long long shape[4], long long stride[4]) {
    if (B < 1 || B > 64 || i < 0 || i > 14) return DBOA_ERR_ARG;
    const Net& n = net();
    const Tape& t = tape_for(B);
    for (int k = 0; k < 4; ++k) { shape[k] = 1; stride[k] = 1; }
    if (i <= 4) {
        int ci = 0;
        bool post = i > 0;
        if (i > 0) {
            int blk = -1;
            for (int l = 0; l < i; ++l) blk += kBlocks[l];
            ci = n.blocks[blk].c3;
        }
        const ConvLayer& c = n.convs[ci];
        *off = post ? t.conv[ci].a : t.conv[ci].y;
        *ndim = 4;
        long long H = c.hout, C = c.cout;
        shape[0] = B; shape[1] = C; shape[2] = H; shape[3] = H;
        stride[0] = H * H * C; stride[1] = 1; stride[2] = H * C; stride[3] = C;
    } else if (i == 5) {
        *off = t.xc; *ndim = 2; shape[0] = B; shape[1] = 2048; stride[0] = HEAD_LD; stride[1] = 1;
    } else {
        int it = (i - 6) / 3, which = (i - 6) % 3;
        long long base = which == 0 ? t.h1pre : (which == 1 ? t.h1post : t.h2pre);
        *off = base + (long long)it * B * HID; *ndim = 2; shape[0] = B; shape[1] = HID; stride[0] = HID; stride[1] = 1;
    }
    return DBOA_OK;
}

}  // namespace dboa
