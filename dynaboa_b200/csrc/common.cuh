// Shared device helpers and launch plumbing for libdynaboa_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define DBOA_OK 0
#define DBOA_ERR_ARG (-1)
#define DBOA_ERR_SHAPE (-2)
#define DBOA_ERR_CUDA (-3)
#define DBOA_ERR_UNSUPPORTED (-4)

namespace dboa {

extern int g_last_cuda_error;      // set by check_launch (defined in hmr_plan.cu)
extern long long g_launch_count;   // number of kernels this library launched (bench "gpu_launches"; replayed graphs credit theirs)

inline int check_launch() {
    ++g_launch_count;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { g_last_cuda_error = (int)e; return DBOA_ERR_CUDA; }
    return DBOA_OK;
}

#define DBOA_TRY(expr) do { int _s = (expr); if (_s != DBOA_OK) return _s; } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Deterministic block-wide sum (fixed tree); result valid in every thread.  blockDim.x <= 1024.
__device__ __forceinline__ float block_sum(float v, float* smem32) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();                 // protect smem32 reuse across consecutive calls
    if (lane == 0) smem32[wid] = v;
    __syncthreads();
    float r = (lane < nw) ? smem32[lane] : 0.f;
    r = warp_sum(r);
    return r;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// True while `st` is being captured into a CUDA graph (or its state cannot be read).  One-time set-up on the launch path
// (allocations, stream / event creation, function attributes) is refused then with DBOA_ERR_UNSUPPORTED, before anything is
// enqueued: dboa_prepare_graph does it ahead of a capture, as does the first eager call.
inline bool stream_capturing(cudaStream_t st) {
    cudaStreamCaptureStatus s = cudaStreamCaptureStatusNone;
    return cudaStreamIsCapturing(st, &s) != cudaSuccess || s != cudaStreamCaptureStatusNone;
}

// SM count of the current device (queried once per process: one process drives one GPU)
inline int num_sms() {
    static const int n = [] {
        int d = 0, v = 0;
        cudaGetDevice(&d);
        return cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d) == cudaSuccess && v > 0 ? v : 132;
    }();
    return n;
}

// ---- programmatic dependent launch (PDL)
// A kernel launched through launch_ex(..., pdl = true) may be scheduled while its predecessor in the stream is still
// running; it must execute pdl_wait() before it touches anything the predecessor reads or writes (all global memory,
// in practice: first statement), and calls pdl_trigger() right after so that ITS successor can be scheduled in turn.
// At batch 1 every layer is a few-microsecond kernel and the launch + block-scheduling latency between dependent
// kernels is a large part of the step; PDL hides it.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool pdl_enabled();                // hmr_plan.cu: true unless DBOA_PDL=0 in the environment

// Launch with optional thread-block-cluster dimensions and PDL.  Non-portable cluster sizes (9..16) and dynamic shared
// memory above 48 KB are enabled once per kernel function.
template <typename... KArgs, typename... Args>
inline int launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, dim3 cluster, bool pdl, Args... args) {
    const unsigned csize = cluster.x * cluster.y * cluster.z;
    {
        // per kernel FUNCTION (several kernels can share one instantiation of this template): bit 0 = non-portable cluster
        // sizes enabled, bit 1 = large dynamic shared memory enabled
        static const void* seen_fn[64];
        static unsigned seen_bits[64];
        static int n_seen = 0;
        int slot = -1;
        for (int i = 0; i < n_seen; ++i)
            if (seen_fn[i] == (const void*)kernel) slot = i;
        if (slot < 0 && n_seen < 64) { slot = n_seen++; seen_fn[slot] = (const void*)kernel; seen_bits[slot] = 0; }
        const unsigned have = slot >= 0 ? seen_bits[slot] : 0u;
        const unsigned want = (csize > 8 ? 1u : 0u) | (smem > 48 * 1024 ? 2u : 0u);
        if (want & ~have) {
            if (stream_capturing(st)) return DBOA_ERR_UNSUPPORTED;
            cudaError_t e = cudaSuccess;
            if ((want & ~have) & 1u) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
            if (e == cudaSuccess && ((want & ~have) & 2u)) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
            if (e != cudaSuccess) { g_last_cuda_error = (int)e; return DBOA_ERR_CUDA; }
            if (slot >= 0) seen_bits[slot] |= want;
        }
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    unsigned na = 0;
    if (csize > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = cluster.x; attr[na].val.clusterDim.y = cluster.y; attr[na].val.clusterDim.z = cluster.z;
        ++na;
    }
    if (pdl && pdl_enabled()) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attr; cfg.numAttrs = na;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
    ++g_launch_count;
    if (e != cudaSuccess) { g_last_cuda_error = (int)e; return DBOA_ERR_CUDA; }
    return DBOA_OK;
}

}  // namespace dboa
