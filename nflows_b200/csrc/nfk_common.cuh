// Shared host-side helpers of libnfk_sm90.so: error reporting, launch accounting.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/nfk.h"

namespace nfk {

extern thread_local char g_last_error[512];
extern std::atomic<int64_t> g_launch_count;

int fail(int code, const char* fmt, ...);

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(NFK_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    return NFK_OK;
}

// Latch for one-time PER-DEVICE setup (cudaFuncSetAttribute and the like): a process may run flows on several GPUs.
struct DeviceOnce {
    std::atomic<uint64_t> done{0};
    bool pending(int* dev) {
        int d = 0;
        cudaGetDevice(&d);
        *dev = d;
        return ((done.load(std::memory_order_acquire) >> (d & 63)) & 1ull) == 0;
    }
    void mark(int dev) { done.fetch_or(1ull << (dev & 63), std::memory_order_release); }
};

namespace tc {
int sm_count();   // multiprocessors of the current device (nfk_linear_tc.cu)
}

// Lets `kernel` launch with `bytes` of dynamic shared memory: above the default limit of 48 KB it has to opt in.
template <class Kernel>
inline int allow_dynamic_smem(Kernel* kernel, size_t bytes) {
    if (bytes <= 48 * 1024) return NFK_OK;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return fail(NFK_E_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    return NFK_OK;
}

// Sum of every thread's v over the block in one fixed order -- a butterfly in each warp, then the n_warps warp sums in order by
// thread 0, which hands the total to out(t) -- so the result does not depend on timing.  Every thread of the block calls it;
// s_warp holds n_warps floats and may be reused once it returns.
template <class Out>
__device__ __forceinline__ void block_sum_in_order(float v, float* s_warp, int n_warps, Out out) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) s_warp[tid >> 5] = v;
    __syncthreads();
    if (tid == 0) {
        float t = 0.0f;
        for (int w = 0; w < n_warps; ++w) t += s_warp[w];
        out(t);
    }
    __syncthreads();
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

inline bool act_valid(int code) { return code >= NFK_ACT_NONE && code < NFK_ACT_COUNT; }

// The conditioner activation of code `code` (include/nfk.h: NFK_ACT_*); relu is fmaxf(x, 0) as it always was.
__device__ __forceinline__ float nfk_act(int code, float x) {
    switch (code) {
        case NFK_ACT_RELU: return fmaxf(x, 0.0f);
        case NFK_ACT_TANH: return tanhf(x);
        case NFK_ACT_ELU: return x > 0.0f ? x : expm1f(x);
        case NFK_ACT_LEAKY_RELU: return x > 0.0f ? x : 0.01f * x;
        case NFK_ACT_GELU: return 0.5f * x * (1.0f + erff(x * 0.707106781186547524f));
        case NFK_ACT_SILU: return x / (1.0f + expf(-x));
        default: return x;
    }
}

}  // namespace nfk

#define NFK_REQUIRE(cond, ...)                                   \
    do {                                                         \
        if (!(cond)) return nfk::fail(NFK_E_INVALID, __VA_ARGS__); \
    } while (0)
