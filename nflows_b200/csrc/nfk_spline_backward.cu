// Backward of the rational-quadratic coupling epilogue (training): the vector-Jacobian product of nfk_rqs_rows with respect to
// its input and its parameters.  See include/nfk.h (nfk_rqs_rows_backward) for the reference lines it differentiates.
#include <algorithm>

#include "nfk_common.cuh"
#include "rq_spline.cuh"

namespace nfk {

constexpr int kBwdThreads = 128;

// One block = 128 threads = 128 consecutive elements e = row * d_t + j per chunk.  The parameters of a chunk are one contiguous
// run of 128 * M floats: fetched with coalesced 16-byte loads into registers one chunk ahead, parked in shared memory, read back
// one element per thread (stride M words), overwritten there by the element's parameter gradients and written out with
// coalesced 16-byte stores.  Every output element is written once by one thread: no atomics, the result does not depend on
// the launch geometry.
template <int KMAX, bool EXACT>
__global__ void __launch_bounds__(kBwdThreads) rqs_rows_backward_kernel(SplineParams p, int inverse, const float* __restrict__ x,
                                                                        int64_t ldx, const float* __restrict__ params,
                                                                        const float* __restrict__ grad_y, int64_t ldgy,
                                                                        const float* __restrict__ grad_lad,
                                                                        float* __restrict__ grad_x, int64_t ldgx,
                                                                        float* __restrict__ grad_params, int d_t, int64_t n_elem) {
    extern __shared__ __align__(16) float sp[];   // [kBwdThreads * M]: the chunk's parameters, then their gradients
    constexpr int kMaxPrefetch = KMAX <= 16 ? (spline_param_count(KMAX, false) + 3) / 4 : 1;
    const int M = spline_param_count(EXACT ? KMAX : p.num_bins, p.linear_tails);
    const int tid = threadIdx.x;
    const int64_t n_chunks = (n_elem + kBwdThreads - 1) / kBwdThreads;
    // a chunk starts 128 * M floats after the previous one: every chunk is 16-byte aligned when the base is
    const bool vec_in = (reinterpret_cast<uintptr_t>(params) & 15u) == 0;
    const bool vec_out = (reinterpret_cast<uintptr_t>(grad_params) & 15u) == 0;
    const bool use_prefetch = KMAX <= 16 && vec_in;
    const int sh_t = (d_t & (d_t - 1)) == 0 ? 31 - __clz(d_t) : -1;

    float4 pre[kMaxPrefetch];
    auto prefetch = [&](const float* src, int n_f) {
        const float4* src4 = reinterpret_cast<const float4*>(src);
#pragma unroll
        for (int u = 0; u < kMaxPrefetch; ++u) {
            const int i = tid + u * kBwdThreads;
            if (i < (n_f >> 2)) pre[u] = __ldcs(src4 + i);
        }
    };
    auto chunk_floats = [&](int64_t c) { return (int)min((int64_t)kBwdThreads, n_elem - c * kBwdThreads) * M; };

    int64_t c = blockIdx.x;
    if (c < n_chunks && use_prefetch) prefetch(params + c * kBwdThreads * (int64_t)M, chunk_floats(c));
    for (; c < n_chunks; c += gridDim.x) {
        const int64_t e0 = c * kBwdThreads;
        const int cnt = (int)min((int64_t)kBwdThreads, n_elem - e0);
        const int n_f = cnt * M;
        const float* src = params + e0 * M;
        if (use_prefetch) {
            float4* dst4 = reinterpret_cast<float4*>(sp);
#pragma unroll
            for (int u = 0; u < kMaxPrefetch; ++u) {
                const int i = tid + u * kBwdThreads;
                if (i < (n_f >> 2)) dst4[i] = pre[u];
            }
            for (int i = (n_f & ~3) + tid; i < n_f; i += kBwdThreads) sp[i] = __ldcs(src + i);
        } else if (vec_in) {
            const float4* src4 = reinterpret_cast<const float4*>(src);
            for (int i = tid; i < (n_f >> 2); i += kBwdThreads) reinterpret_cast<float4*>(sp)[i] = __ldcs(src4 + i);
            for (int i = (n_f & ~3) + tid; i < n_f; i += kBwdThreads) sp[i] = __ldcs(src + i);
        } else {
            for (int i = tid; i < n_f; i += kBwdThreads) sp[i] = __ldcs(src + i);
        }
        __syncthreads();
        const int64_t nc = c + gridDim.x;
        if (nc < n_chunks && use_prefetch) prefetch(params + nc * kBwdThreads * (int64_t)M, chunk_floats(nc));

        if (tid < cnt) {
            const int64_t e = e0 + tid;
            const int64_t row = sh_t >= 0 ? e >> sh_t : e / d_t;
            const int j = (int)(e - row * d_t);
            float* q = sp + tid * M;
            float w[KMAX], h[KMAX], d[KMAX + 1];
            rqs_load_packed<KMAX, EXACT>(p, [&](int i) { return q[i]; }, w, h, d);
            const float xin = x[row * ldx + j];
            const float gy = grad_y ? grad_y[row * ldgy + j] : 0.0f;
            const float gl = grad_lad ? __ldg(grad_lad + row) : 0.0f;
            float gx;
            // the EXACT instances pair with the lean forward form (rqs_eval_lean): the same knot arithmetic finds the same bin
            rqs_vjp<KMAX, EXACT, EXACT>(p, inverse != 0, xin, w, h, d, gy, gl, gx);
            rqs_store_grads<KMAX, EXACT>(p, w, h, d, [&](int i, float g) { q[i] = g; });
            if (grad_x) grad_x[row * ldgx + j] = gx;
        }
        __syncthreads();
        float* dst = grad_params + e0 * M;
        if (vec_out) {
            for (int i = tid; i < (n_f >> 2); i += kBwdThreads) __stcs(reinterpret_cast<float4*>(dst) + i, reinterpret_cast<float4*>(sp)[i]);
            for (int i = (n_f & ~3) + tid; i < n_f; i += kBwdThreads) dst[i] = sp[i];
        } else {
            for (int i = tid; i < n_f; i += kBwdThreads) dst[i] = sp[i];
        }
        __syncthreads();
    }
}

template <int KMAX, bool EXACT>
static int launch_rows_backward(const SplineParams& p, int inverse, const float* x, int64_t ldx, const float* params,
                                const float* grad_y, int64_t ldgy, const float* grad_lad, float* grad_x, int64_t ldgx,
                                float* grad_params, int d_t, int64_t n_elem, cudaStream_t st) {
    const size_t smem = (size_t)kBwdThreads * spline_param_count(p.num_bins, p.linear_tails) * sizeof(float);
    if (int rc = allow_dynamic_smem(rqs_rows_backward_kernel<KMAX, EXACT>, smem)) return rc;
    const int64_t n_chunks = (n_elem + kBwdThreads - 1) / kBwdThreads;
    const int grid = (int)std::min<int64_t>(n_chunks, (int64_t)tc::sm_count() * 32);
    rqs_rows_backward_kernel<KMAX, EXACT><<<grid, kBwdThreads, smem, st>>>(p, inverse, x, ldx, params, grad_y, ldgy, grad_lad,
                                                                          grad_x, ldgx, grad_params, d_t, n_elem);
    return check_launch("rqs_rows_backward_kernel");
}

}  // namespace nfk

using namespace nfk;

extern "C" int nfk_rqs_rows_backward(const NfkSplineDesc* desc, int inverse, const float* x, int64_t ldx, const float* params,
                                     const float* grad_y, int64_t ldgy, const float* grad_lad, float* grad_x, int64_t ldgx,
                                     float* grad_params, int32_t d_t, int64_t n_rows, void* stream) {
    SplineParams p;
    int rc = make_spline_params(desc, &p);
    if (rc) return rc;
    NFK_REQUIRE(n_rows >= 0 && d_t >= 1, "bad sizes n_rows=%lld d_t=%d", (long long)n_rows, d_t);
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(x && params && grad_params, "NULL tensor pointer");
    NFK_REQUIRE(ldx >= d_t && (!grad_y || ldgy >= d_t) && (!grad_x || ldgx >= d_t),
                "row strides must be >= d_t=%d (ldx=%lld ldgy=%lld ldgx=%lld)", d_t, (long long)ldx, (long long)ldgy,
                (long long)ldgx);
    NFK_REQUIRE(grad_params != params, "grad_params must not alias params");
    NFK_REQUIRE(!grad_x || (grad_x != x && (const float*)grad_x != grad_y), "grad_x must not alias x or grad_y");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n_elem = n_rows * d_t;
    return with_bin_instance(p.num_bins, [&](auto km, auto ex) {
        return launch_rows_backward<km, ex>(p, inverse, x, ldx, params, grad_y, ldgy, grad_lad, grad_x, ldgx, grad_params, d_t, n_elem,
                                            st);
    });
}
