// Rational-quadratic spline on the plane layout of image couplings (forward and backward), and the backward of the spline whose
// parameters the whole batch shares (PiecewiseRationalQuadraticCDF).  See include/nfk.h (nfk_rqs_planes, nfk_rqs_planes_backward,
// nfk_rqs_shared_backward) for the reference lines each one replaces.
#include <algorithm>

#include "nfk_common.cuh"
#include "rq_spline.cuh"

namespace nfk {

// ------------------------------------------------------------------------------------------------------------------------
// plane layout: element (b, j, p) of x at x[b*ldx + j*P + p], its parameter k at params[b*ldp + (j*M + k)*P + p]
// ------------------------------------------------------------------------------------------------------------------------
// One block per sample (grid-stride over samples), thread t takes the sample's elements e = j*P + p = t, t + T, ... in that order.
// The block size T depends on C_t*P alone, so each sample's log|det| is summed in one fixed order (per thread, then a shuffle
// butterfly, then the warps in order) whatever the batch, its split or the grid: bitwise reproducible.
// Parameters are read straight from global memory, not staged: a sample's C_t*M*P parameters are one contiguous run that the block
// reads completely, so for P < 32 the 32-byte sectors a warp touches for parameter k are finished by its reads of parameter k + 1
// out of L1 (the loads are L1-cached, the run of a block stays resident while it is consumed).  Staging the run in shared memory
// would cost 4*C_t*M*P bytes per sample (141 KB at level 1 of cfg 5) or chunking by elements that are not contiguous in memory.
constexpr int kPlanesMaxThreads = 256;

inline int planes_threads(int64_t n_el) {
    return (int)std::min<int64_t>(kPlanesMaxThreads, std::max<int64_t>(32, (n_el + 31) / 32 * 32));
}

template <int KMAX, bool EXACT>
__device__ __forceinline__ void planes_load(const SplineParams& p, const float* __restrict__ q, int64_t P, float (&w)[KMAX],
                                            float (&h)[KMAX], float (&d)[KMAX + 1]) {
    const int K = EXACT ? KMAX : p.num_bins;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        w[k] = (k < K) ? __ldg(q + k * P) : 0.0f;
        h[k] = (k < K) ? __ldg(q + (K + k) * P) : 0.0f;
    }
    if (p.linear_tails) {
#pragma unroll
        for (int k = 0; k <= KMAX; ++k) d[k] = (k >= 1 && k < K) ? __ldg(q + (2 * K + k - 1) * P) : p.edge_ud;
    } else {
#pragma unroll
        for (int k = 0; k <= KMAX; ++k) d[k] = (k <= K) ? __ldg(q + (2 * K + k) * P) : 0.0f;
    }
}

template <int KMAX, bool EXACT>
__global__ void __launch_bounds__(kPlanesMaxThreads) rqs_planes_kernel(SplineParams p, int inverse, const float* __restrict__ x,
                                                                       int64_t ldx, const float* __restrict__ params, int64_t ldp,
                                                                       int c_t, int P, float* __restrict__ y, int64_t ldy,
                                                                       float* __restrict__ lad_accum, int64_t n_samples,
                                                                       int32_t* flags) {
    __shared__ float s_lad[kPlanesMaxThreads / 32];
    const int K = EXACT ? KMAX : p.num_bins;
    const int M = p.linear_tails ? 3 * K - 1 : 3 * K + 1;
    const int n_el = c_t * P;
    const int tid = threadIdx.x;
    int flag = 0;
    for (int64_t b = blockIdx.x; b < n_samples; b += gridDim.x) {
        float my_lad = 0.0f;
        for (int e = tid; e < n_el; e += blockDim.x) {
            const int j = e / P, px = e - j * P;
            const float* q = params + b * ldp + (int64_t)j * M * P + px;
            const float xin = x[b * ldx + e];
            float yy, ll;
            if (EXACT) {
                // the lean form on the same registers the EXACT instances of nfk_rqs_rows use
                constexpr int MPL = 3 * KMAX + 1;
                float v[MPL];
                const float xi[1] = {xin};
                float y1[1], l1[1];
                if (p.linear_tails) {
#pragma unroll
                    for (int k = 0; k < 3 * KMAX - 1; ++k) v[k] = __ldg(q + (int64_t)k * P);
                    if (inverse) rqs_eval_lean<KMAX, true, true, 1, MPL>(p, xi, v, y1, l1, flag);
                    else rqs_eval_lean<KMAX, true, false, 1, MPL>(p, xi, v, y1, l1, flag);
                } else {
#pragma unroll
                    for (int k = 0; k < 3 * KMAX + 1; ++k) v[k] = __ldg(q + (int64_t)k * P);
                    if (inverse) rqs_eval_lean<KMAX, false, true, 1, MPL>(p, xi, v, y1, l1, flag);
                    else rqs_eval_lean<KMAX, false, false, 1, MPL>(p, xi, v, y1, l1, flag);
                }
                yy = y1[0];
                ll = l1[0];
            } else {
                float w[KMAX], h[KMAX], d[KMAX + 1];
                planes_load<KMAX, EXACT>(p, q, P, w, h, d);
                rqs_eval<KMAX, EXACT>(p, inverse != 0, xin, w, h, d, yy, ll, flag);
            }
            y[b * ldy + e] = yy;
            my_lad += ll;
        }
        if (lad_accum) {
            float v = my_lad;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if ((tid & 31) == 0) s_lad[tid >> 5] = v;
            __syncthreads();
            if (tid == 0) {
                float t = 0.0f;
                for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_lad[w];
                lad_accum[b] += t;
            }
            __syncthreads();
        }
    }
    if (flag && flags) atomicOr(flags, flag);
}

// The backward: one thread per element, every output entry written once by the thread of its element (no reduction, so the
// launch geometry does not matter).  A thread parks its element's M parameters in its own run of shared memory (stride M words) and
// evaluates the VJP on them as nfk_rqs_rows_backward does on its staged chunk: with the parameters read through 64-bit strided
// addresses instead, the KMAX = 64 instance spilled.
constexpr int kPlanesBwdThreads = 128;

template <int KMAX, bool EXACT>
__global__ void __launch_bounds__(kPlanesBwdThreads) rqs_planes_backward_kernel(
    SplineParams p, int inverse, const float* __restrict__ x, int64_t ldx, const float* __restrict__ params, int64_t ldp,
    const float* __restrict__ grad_y, int64_t ldgy, const float* __restrict__ grad_lad, float* __restrict__ grad_x, int64_t ldgx,
    float* __restrict__ grad_params, int64_t ldgp, int c_t, int P, int64_t n_samples) {
    extern __shared__ float sp[];      // [kPlanesBwdThreads * M]: thread t's element at sp[t*M ..)
    const int K = EXACT ? KMAX : p.num_bins;
    const int M = p.linear_tails ? 3 * K - 1 : 3 * K + 1;
    const int64_t n_el = (int64_t)c_t * P;
    float* q = sp + threadIdx.x * M;
    for (int64_t i = (int64_t)blockIdx.x * kPlanesBwdThreads + threadIdx.x; i < n_samples * n_el;
         i += (int64_t)gridDim.x * kPlanesBwdThreads) {
        const int64_t b = i / n_el;
        const int e = (int)(i - b * n_el);
        const int j = e / P, px = e - j * P;
        const int64_t off = (int64_t)j * M * P + px;
        const float* src = params + b * ldp + off;
        for (int k = 0; k < M; ++k) q[k] = __ldg(src + (int64_t)k * P);
        float w[KMAX], h[KMAX], d[KMAX + 1];
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            w[k] = (k < K) ? q[k] : 0.0f;
            h[k] = (k < K) ? q[K + k] : 0.0f;
        }
        if (p.linear_tails) {
#pragma unroll
            for (int k = 0; k <= KMAX; ++k) d[k] = (k >= 1 && k < K) ? q[2 * K + k - 1] : p.edge_ud;
        } else {
#pragma unroll
            for (int k = 0; k <= KMAX; ++k) d[k] = (k <= K) ? q[2 * K + k] : 0.0f;
        }
        const float gy = grad_y ? grad_y[b * ldgy + e] : 0.0f;
        const float gl = grad_lad ? __ldg(grad_lad + b) : 0.0f;
        float gx;
        // the EXACT instances pair with the lean forward form (rqs_eval_lean): the same knot arithmetic finds the same bin
        rqs_vjp<KMAX, EXACT, EXACT>(p, inverse != 0, x[b * ldx + e], w, h, d, gy, gl, gx);
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            if (k < K) {
                q[k] = w[k];
                q[K + k] = h[k];
            }
        }
        if (p.linear_tails) {
#pragma unroll
            for (int k = 1; k < KMAX; ++k)
                if (k < K) q[2 * K + k - 1] = d[k];
        } else {
#pragma unroll
            for (int k = 0; k <= KMAX; ++k)
                if (k <= K) q[2 * K + k] = d[k];
        }
        float* dst = grad_params + b * ldgp + off;
        for (int k = 0; k < M; ++k) __stcs(dst + (int64_t)k * P, q[k]);
        if (grad_x) grad_x[b * ldgx + e] = gx;
    }
}

template <int KMAX, bool EXACT>
static int launch_planes(const SplineParams& p, int inverse, const float* x, int64_t ldx, const float* params, int64_t ldp, int c_t,
                         int P, float* y, int64_t ldy, float* lad_accum, int64_t n_samples, int32_t* flags, cudaStream_t st) {
    const int threads = planes_threads((int64_t)c_t * P);
    const int grid = (int)std::min<int64_t>(n_samples, (int64_t)tc::sm_count() * (2048 / threads));
    rqs_planes_kernel<KMAX, EXACT><<<grid, threads, 0, st>>>(p, inverse, x, ldx, params, ldp, c_t, P, y, ldy, lad_accum, n_samples,
                                                            flags);
    return check_launch("rqs_planes_kernel");
}

template <int KMAX, bool EXACT>
static int launch_planes_backward(const SplineParams& p, int inverse, const float* x, int64_t ldx, const float* params, int64_t ldp,
                                  const float* grad_y, int64_t ldgy, const float* grad_lad, float* grad_x, int64_t ldgx,
                                  float* grad_params, int64_t ldgp, int c_t, int P, int64_t n_samples, cudaStream_t st) {
    const int M = p.linear_tails ? 3 * p.num_bins - 1 : 3 * p.num_bins + 1;
    const size_t smem = (size_t)kPlanesBwdThreads * M * sizeof(float);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(rqs_planes_backward_kernel<KMAX, EXACT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem);
        if (e != cudaSuccess) return fail(NFK_E_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    }
    const int64_t n_blocks = (n_samples * c_t * P + kPlanesBwdThreads - 1) / kPlanesBwdThreads;
    const int grid = (int)std::min<int64_t>(n_blocks, (int64_t)tc::sm_count() * 32);
    rqs_planes_backward_kernel<KMAX, EXACT><<<grid, kPlanesBwdThreads, smem, st>>>(p, inverse, x, ldx, params, ldp, grad_y, ldgy,
                                                                                  grad_lad, grad_x, ldgx, grad_params, ldgp, c_t, P,
                                                                                  n_samples);
    return check_launch("rqs_planes_backward_kernel");
}

// ------------------------------------------------------------------------------------------------------------------------
// batch-shared parameters: x [B, F], uw / uh [F, K], ud [F, K -+ 1]; parameter gradients summed over the batch
// ------------------------------------------------------------------------------------------------------------------------
// Pass 1: thread (s, f) runs the VJP of feature f over the S rows of slab s in row order and keeps the running parameter sums in
// shared memory (entry k of thread t at [k*T + t]: conflict-free); it writes them to ws[(s*MT + k)*F + f] (MT = 2K + number of
// derivatives), coalesced over f.  Pass 2: one block per 32 consecutive entries (k, f) of the result, warp w sums a contiguous
// range of slabs in order, lane l's 32 warp sums are added in order.  S depends only on (B, F) and is at most 256 rows, so every
// fp32 sum runs over at most 256 terms (slab), 2048 terms (a warp's slabs at B = 2^20) and 32 terms (warps).
constexpr int kSharedThreads = 64;
constexpr int kSharedMaxSlab = 256;
constexpr int kSumWarps = 32;

inline int shared_slab_rows(int64_t n_rows, int64_t F) {
    // enough (slab, feature) threads to fill an H100 (~2^17) where the batch allows, slabs of 16 .. 256 rows
    int s = kSharedMaxSlab;
    while (s > 16 && n_rows * F / s < (1 << 17)) s >>= 1;
    return s;
}

inline int shared_mt(int K, int linear_tails) { return 2 * K + (linear_tails ? K - 1 : K + 1); }

// The feature's raw parameters are parked once in shared memory next to the running sums (thread t's entry k at [k*T + t]) and
// read back for every row: the VJP overwrites its register copies, and a second register copy spilled at KMAX = 64.
template <int KMAX, bool EXACT>
__global__ void __launch_bounds__(kSharedThreads) rqs_shared_backward_kernel(
    SplineParams p, int inverse, const float* __restrict__ x, const float* __restrict__ uw, const float* __restrict__ uh,
    const float* __restrict__ ud, const float* __restrict__ grad_y, const float* __restrict__ grad_lad, float* __restrict__ grad_x,
    float* __restrict__ ws, int F, int64_t n_rows, int slab, int64_t n_slabs) {
    extern __shared__ float sm[];      // [MT][kSharedThreads] parameters, then [MT][kSharedThreads] sums
    const int K = EXACT ? KMAX : p.num_bins;
    const int nd = p.linear_tails ? K - 1 : K + 1;
    const int MT = 2 * K + nd;
    const int tid = threadIdx.x;
    const int64_t t = (int64_t)blockIdx.x * kSharedThreads + tid;
    if (t >= n_slabs * F) return;
    const int64_t s = t / F;
    const int f = (int)(t - s * F);
    float* par = sm + tid;
    float* acc = sm + MT * kSharedThreads + tid;
    for (int k = 0; k < K; ++k) {
        par[k * kSharedThreads] = __ldg(uw + (int64_t)f * K + k);
        par[(K + k) * kSharedThreads] = __ldg(uh + (int64_t)f * K + k);
    }
    for (int k = 0; k < nd; ++k) par[(2 * K + k) * kSharedThreads] = __ldg(ud + (int64_t)f * nd + k);
    for (int k = 0; k < MT; ++k) acc[k * kSharedThreads] = 0.0f;
    const int64_t r0 = s * slab, r1 = min(n_rows, r0 + slab);
    for (int64_t r = r0; r < r1; ++r) {
        float w[KMAX], h[KMAX], d[KMAX + 1];
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            w[k] = (k < K) ? par[k * kSharedThreads] : 0.0f;
            h[k] = (k < K) ? par[(K + k) * kSharedThreads] : 0.0f;
        }
        if (p.linear_tails) {
#pragma unroll
            for (int k = 0; k <= KMAX; ++k) d[k] = (k >= 1 && k < K) ? par[(2 * K + k - 1) * kSharedThreads] : p.edge_ud;
        } else {
#pragma unroll
            for (int k = 0; k <= KMAX; ++k) d[k] = (k <= K) ? par[(2 * K + k) * kSharedThreads] : 0.0f;
        }
        const int64_t e = r * F + f;
        const float gy = grad_y ? __ldcs(grad_y + e) : 0.0f;
        const float gl = grad_lad ? __ldg(grad_lad + r) : 0.0f;
        float gx;
        // nfk_rqs_elementwise evaluates the scan form (rqs_eval) at every instance: LEAN = false finds its bin
        rqs_vjp<KMAX, EXACT, false>(p, inverse != 0, __ldcs(x + e), w, h, d, gy, gl, gx);
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
            if (k < K) {
                acc[k * kSharedThreads] += w[k];
                acc[(K + k) * kSharedThreads] += h[k];
            }
        }
        if (p.linear_tails) {
#pragma unroll
            for (int k = 1; k < KMAX; ++k)
                if (k < K) acc[(2 * K + k - 1) * kSharedThreads] += d[k];
        } else {
#pragma unroll
            for (int k = 0; k <= KMAX; ++k)
                if (k <= K) acc[(2 * K + k) * kSharedThreads] += d[k];
        }
        if (grad_x) __stcs(grad_x + e, gx);
    }
    for (int k = 0; k < MT; ++k) ws[(s * MT + k) * F + f] = acc[k * kSharedThreads];
}

// result entry i = k*F + f (k < MT) -> grad_uw[f*K + k], grad_uh[f*K + k - K] or grad_ud[f*nd + k - 2K]
__global__ void __launch_bounds__(kSumWarps * 32) rqs_shared_sum_kernel(const float* __restrict__ ws, int64_t n_entries,
                                                                        int64_t n_slabs, int F, int K, int nd,
                                                                        float* __restrict__ grad_uw, float* __restrict__ grad_uh,
                                                                        float* __restrict__ grad_ud) {
    __shared__ float part[kSumWarps][33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t i = (int64_t)blockIdx.x * 32 + lane;
    const int64_t per = (n_slabs + kSumWarps - 1) / kSumWarps;
    const int64_t s0 = warp * per, s1 = min(n_slabs, s0 + per);
    float v = 0.0f;
    if (i < n_entries)
        for (int64_t s = s0; s < s1; ++s) v += __ldcs(ws + s * n_entries + i);
    part[warp][lane] = v;
    __syncthreads();
    if (warp == 0 && i < n_entries) {
        float t = 0.0f;
        for (int w = 0; w < kSumWarps; ++w) t += part[w][lane];
        const int k = (int)(i / F), f = (int)(i - (int64_t)k * F);
        if (k < K) grad_uw[(int64_t)f * K + k] = t;
        else if (k < 2 * K) grad_uh[(int64_t)f * K + k - K] = t;
        else grad_ud[(int64_t)f * nd + k - 2 * K] = t;
    }
}

template <int KMAX, bool EXACT>
static int launch_shared_backward(const SplineParams& p, int inverse, const float* x, const float* uw, const float* uh,
                                  const float* ud, const float* grad_y, const float* grad_lad, float* grad_x, float* grad_uw,
                                  float* grad_uh, float* grad_ud, int F, int64_t n_rows, float* ws, cudaStream_t st) {
    const int K = p.num_bins;
    const int nd = p.linear_tails ? K - 1 : K + 1;
    const int MT = 2 * K + nd;
    const int slab = shared_slab_rows(n_rows, F);
    const int64_t n_slabs = (n_rows + slab - 1) / slab;
    const size_t smem = (size_t)2 * MT * kSharedThreads * sizeof(float);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(rqs_shared_backward_kernel<KMAX, EXACT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem);
        if (e != cudaSuccess) return fail(NFK_E_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    }
    const int64_t n_threads = n_slabs * F;
    const int64_t grid1 = (n_threads + kSharedThreads - 1) / kSharedThreads;
    rqs_shared_backward_kernel<KMAX, EXACT><<<(unsigned)grid1, kSharedThreads, smem, st>>>(
        p, inverse, x, uw, uh, ud, grad_y, grad_lad, grad_x, ws, F, n_rows, slab, n_slabs);
    int rc = check_launch("rqs_shared_backward_kernel");
    if (rc) return rc;
    const int64_t n_entries = (int64_t)MT * F;
    rqs_shared_sum_kernel<<<(unsigned)((n_entries + 31) / 32), kSumWarps * 32, 0, st>>>(ws, n_entries, n_slabs, F, K, nd, grad_uw,
                                                                                        grad_uh, grad_ud);
    return check_launch("rqs_shared_sum_kernel");
}

static bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
    const char* pa = static_cast<const char*>(a);
    const char* pb = static_cast<const char*>(b);
    return a && b && na && nb && pa < pb + nb && pb < pa + na;
}

}  // namespace nfk

using namespace nfk;

extern "C" int nfk_rqs_planes(const NfkSplineDesc* desc, int inverse, const float* x, int64_t ldx, const float* params, int64_t ldp,
                              int32_t c_t, int32_t pixels, float* y, int64_t ldy, float* lad_accum, int64_t n_samples,
                              int32_t* flags, void* stream) {
    SplineParams p;
    int rc = make_spline_params(desc, &p);
    if (rc) return rc;
    NFK_REQUIRE(n_samples >= 0 && c_t >= 1 && pixels >= 1, "bad sizes n_samples=%lld c_t=%d pixels=%d", (long long)n_samples, c_t,
                pixels);
    const int64_t M = p.linear_tails ? 3 * p.num_bins - 1 : 3 * p.num_bins + 1;
    NFK_REQUIRE((int64_t)c_t * M * pixels <= INT32_MAX, "a sample's %lld parameters exceed the 32-bit element index",
                (long long)((int64_t)c_t * M * pixels));
    if (n_samples == 0) return NFK_OK;
    NFK_REQUIRE(x && params && y, "NULL tensor pointer");
    const int64_t n_el = (int64_t)c_t * pixels;
    NFK_REQUIRE(ldx >= n_el && ldy >= n_el && ldp >= n_el * M,
                "sample strides too small (ldx=%lld ldy=%lld >= %lld, ldp=%lld >= %lld)", (long long)ldx, (long long)ldy,
                (long long)n_el, (long long)ldp, (long long)(n_el * M));
    NFK_REQUIRE(x != y && (const float*)y != params, "y must not alias x or params");
    cudaStream_t st = (cudaStream_t)stream;
#define NFK_PLANES(KM, EX) \
    return launch_planes<KM, EX>(p, inverse, x, ldx, params, ldp, c_t, pixels, y, ldy, lad_accum, n_samples, flags, st)
    if (p.num_bins == 8) NFK_PLANES(8, true);
    if (p.num_bins < 8) NFK_PLANES(8, false);
    if (p.num_bins == 16) NFK_PLANES(16, true);
    if (p.num_bins < 16) NFK_PLANES(16, false);
    if (p.num_bins <= 32) NFK_PLANES(32, false);
    NFK_PLANES(64, false);
#undef NFK_PLANES
}

extern "C" int nfk_rqs_planes_backward(const NfkSplineDesc* desc, int inverse, const float* x, int64_t ldx, const float* params,
                                       int64_t ldp, const float* grad_y, int64_t ldgy, const float* grad_lad, float* grad_x,
                                       int64_t ldgx, float* grad_params, int64_t ldgp, int32_t c_t, int32_t pixels,
                                       int64_t n_samples, void* stream) {
    SplineParams p;
    int rc = make_spline_params(desc, &p);
    if (rc) return rc;
    NFK_REQUIRE(n_samples >= 0 && c_t >= 1 && pixels >= 1, "bad sizes n_samples=%lld c_t=%d pixels=%d", (long long)n_samples, c_t,
                pixels);
    const int64_t M = p.linear_tails ? 3 * p.num_bins - 1 : 3 * p.num_bins + 1;
    NFK_REQUIRE((int64_t)c_t * M * pixels <= INT32_MAX, "a sample's %lld parameters exceed the 32-bit element index",
                (long long)((int64_t)c_t * M * pixels));
    if (n_samples == 0) return NFK_OK;
    NFK_REQUIRE(x && params && grad_params, "NULL tensor pointer");
    const int64_t n_el = (int64_t)c_t * pixels;
    NFK_REQUIRE(ldx >= n_el && (!grad_y || ldgy >= n_el) && (!grad_x || ldgx >= n_el) && ldp >= n_el * M && ldgp >= n_el * M,
                "sample strides too small (ldx=%lld ldgy=%lld ldgx=%lld >= %lld, ldp=%lld ldgp=%lld >= %lld)", (long long)ldx,
                (long long)ldgy, (long long)ldgx, (long long)n_el, (long long)ldp, (long long)ldgp, (long long)(n_el * M));
    NFK_REQUIRE(grad_params != params, "grad_params must not alias params");
    NFK_REQUIRE(!grad_x || (grad_x != x && (const float*)grad_x != grad_y), "grad_x must not alias x or grad_y");
    cudaStream_t st = (cudaStream_t)stream;
#define NFK_PLANES_BWD(KM, EX)                                                                                                  \
    return launch_planes_backward<KM, EX>(p, inverse, x, ldx, params, ldp, grad_y, ldgy, grad_lad, grad_x, ldgx, grad_params, ldgp, \
                                          c_t, pixels, n_samples, st)
    if (p.num_bins == 8) NFK_PLANES_BWD(8, true);
    if (p.num_bins < 8) NFK_PLANES_BWD(8, false);
    if (p.num_bins == 16) NFK_PLANES_BWD(16, true);
    if (p.num_bins < 16) NFK_PLANES_BWD(16, false);
    if (p.num_bins <= 32) NFK_PLANES_BWD(32, false);
    NFK_PLANES_BWD(64, false);
#undef NFK_PLANES_BWD
}

extern "C" size_t nfk_rqs_shared_backward_workspace(int64_t n_rows, int32_t features, int32_t num_bins, int32_t linear_tails) {
    if (n_rows <= 0 || features <= 0 || num_bins < 1 || num_bins > NFK_MAX_BINS) return 0;
    const int64_t slab = shared_slab_rows(n_rows, features);
    const int64_t n_slabs = (n_rows + slab - 1) / slab;
    return (size_t)(n_slabs * shared_mt(num_bins, linear_tails) * features) * sizeof(float);
}

extern "C" int nfk_rqs_shared_backward(const NfkSplineDesc* desc, int inverse, const float* x, const float* uw, const float* uh,
                                       const float* ud, const float* grad_y, const float* grad_lad, float* grad_x, float* grad_uw,
                                       float* grad_uh, float* grad_ud, int32_t features, int64_t n_rows, void* workspace,
                                       size_t workspace_bytes, void* stream) {
    SplineParams p;
    int rc = make_spline_params(desc, &p);
    if (rc) return rc;
    NFK_REQUIRE(n_rows >= 0 && features >= 1, "bad sizes n_rows=%lld features=%d", (long long)n_rows, features);
    const int K = p.num_bins;
    const int nd = p.linear_tails ? K - 1 : K + 1;
    // one bin with linear tails has no interior derivative: an empty ud / grad_ud may be NULL
    NFK_REQUIRE(uw && uh && (ud || nd == 0) && grad_uw && grad_uh && (grad_ud || nd == 0), "NULL parameter pointer");
    if (n_rows == 0) {
        // no rows: every parameter gradient is a sum of nothing
        cudaStream_t st = (cudaStream_t)stream;
        const size_t fk = (size_t)features * K * sizeof(float);
        cudaError_t e = cudaMemsetAsync(grad_uw, 0, fk, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(grad_uh, 0, fk, st);
        if (e == cudaSuccess && nd) e = cudaMemsetAsync(grad_ud, 0, (size_t)features * nd * sizeof(float), st);
        if (e != cudaSuccess) return fail(NFK_E_CUDA, "cudaMemsetAsync: %s", cudaGetErrorString(e));
        return NFK_OK;
    }
    NFK_REQUIRE(x, "NULL tensor pointer");
    const size_t need = nfk_rqs_shared_backward_workspace(n_rows, features, K, p.linear_tails);
    NFK_REQUIRE(workspace && workspace_bytes >= need, "workspace of %zu bytes, need %zu (nfk_rqs_shared_backward_workspace)",
                workspace_bytes, need);
    const size_t xb = (size_t)n_rows * features * sizeof(float);
    const size_t kb = (size_t)features * K * sizeof(float), db = (size_t)features * nd * sizeof(float);
    NFK_REQUIRE(!grad_x || (!overlaps(grad_x, xb, x, xb) && !overlaps(grad_x, xb, grad_y, xb)), "grad_x must not alias x or grad_y");
    const void* outs[3] = {grad_uw, grad_uh, grad_ud};
    const size_t out_b[3] = {kb, kb, db};
    const void* ins[5] = {x, uw, uh, ud, workspace};
    const size_t in_b[5] = {xb, kb, kb, db, need};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 5; ++j) NFK_REQUIRE(!overlaps(outs[i], out_b[i], ins[j], in_b[j]), "parameter gradients must not alias inputs or the workspace");
        for (int j = 0; j < i; ++j) NFK_REQUIRE(!overlaps(outs[i], out_b[i], outs[j], out_b[j]), "parameter gradients must not alias each other");
        NFK_REQUIRE(!overlaps(outs[i], out_b[i], grad_x, xb), "parameter gradients must not alias grad_x");
    }
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = static_cast<float*>(workspace);
#define NFK_SHARED_BWD(KM, EX)                                                                                                      \
    return launch_shared_backward<KM, EX>(p, inverse, x, uw, uh, ud, grad_y, grad_lad, grad_x, grad_uw, grad_uh, grad_ud, features, \
                                          n_rows, ws, st)
    if (K == 8) NFK_SHARED_BWD(8, true);
    if (K < 8) NFK_SHARED_BWD(8, false);
    if (K == 16) NFK_SHARED_BWD(16, true);
    if (K < 16) NFK_SHARED_BWD(16, false);
    if (K <= 32) NFK_SHARED_BWD(32, false);
    NFK_SHARED_BWD(64, false);
#undef NFK_SHARED_BWD
}
