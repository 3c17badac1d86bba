// Row-wise elementwise kernels of the path: column gather (identity split / Permutation), ActNorm, affine and
// additive coupling epilogues, StandardNormal log-density, log|det| bookkeeping.  All HBM-bound; one pass each.
#include <math.h>

#include "nfk_common.cuh"

namespace nfk {

constexpr int kThreads = 256;

static inline int grid_for(int64_t work_items, int threads) {
    int64_t g = (work_items + threads - 1) / threads;
    const int64_t cap = (int64_t)nfk::tc::sm_count() * 64;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

__global__ void __launch_bounds__(kThreads) gather_cols_kernel(const float* __restrict__ x, int64_t ldx,
                                                               const int32_t* __restrict__ cols, int n_cols,
                                                               float* __restrict__ out, int64_t ldo, int64_t n_rows) {
    const int64_t total = n_rows * n_cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / n_cols;
        const int j = (int)(i - r * n_cols);
        out[r * ldo + j] = x[r * ldx + __ldg(cols + j)];
    }
}

__global__ void __launch_bounds__(kThreads) actnorm_kernel(const float* __restrict__ x, int64_t ldx,
                                                           const float* __restrict__ scale,
                                                           const float* __restrict__ shift, float* __restrict__ y,
                                                           int64_t ldy, float* __restrict__ lad_accum, float lad_const,
                                                           int64_t n_rows, int d, int inverse) {
    const int64_t total = n_rows * d;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / d;
        const int j = (int)(i - r * d);
        const float v = x[r * ldx + j];
        const float s = __ldg(scale + j), t = __ldg(shift + j);
        // forward: scale * inputs + shift (two roundings, like the reference's mul then add); inverse: (x - shift) / scale
        y[r * ldy + j] = inverse ? __fdiv_rn(__fsub_rn(v, t), s) : __fadd_rn(__fmul_rn(s, v), t);
        if (j == 0 && lad_accum) lad_accum[r] += lad_const;
    }
}

__global__ void __launch_bounds__(kThreads) add_const_kernel(float* __restrict__ a, float c, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] += c;
}

__global__ void __launch_bounds__(kThreads) fill_kernel(float* __restrict__ a, float c, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] = c;
}

__device__ __forceinline__ float sigmoid_torch(float v) { return 1.0f / (1.0f + expf(-v)); }

// one warp per row; lanes stride over the transformed features; fixed-order warp reduction of log(scale)
__global__ void __launch_bounds__(kThreads) affine_coupling_rows_kernel(
    const float* __restrict__ x, int64_t ldx, const float* __restrict__ params, int mult, int scale_activation, int inverse,
    const int32_t* __restrict__ t_cols, int d_t, const int32_t* __restrict__ id_cols, int d_id, float* __restrict__ y,
    int64_t ldy, float* __restrict__ lad_accum, int64_t n_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp0; r < n_rows; r += n_warps) {
        const float* pr = params + r * (int64_t)mult * d_t;
        float acc = 0.0f;
        for (int j = lane; j < d_t; j += 32) {
            const int col = t_cols ? __ldg(t_cols + j) : j;
            const float v = x[r * ldx + col];
            const float shift = pr[j];
            float out;
            if (mult == 2) {
                const float u = pr[d_t + j];
                float scale;
                if (scale_activation == 0) {
                    scale = sigmoid_torch(u + 2.0f) + 1e-3f;
                } else {
                    float sp = u > 20.0f ? u : log1pf(expf(u));
                    scale = fminf(fmaxf(sp + 1e-3f, 0.0f), 3.0f);
                }
                acc += logf(scale);
                out = inverse ? __fdiv_rn(__fsub_rn(v, shift), scale) : __fadd_rn(__fmul_rn(v, scale), shift);
            } else {
                out = inverse ? (v - shift) : (v + shift);   // additive: scale == 1 exactly, log|det| == 0
            }
            y[r * ldy + col] = out;
        }
        for (int j = lane; j < d_id; j += 32) {
            const int col = __ldg(id_cols + j);
            y[r * ldy + col] = x[r * ldx + col];
        }
        if (lad_accum && mult == 2) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) lad_accum[r] += inverse ? -acc : acc;
        }
    }
}

__global__ void __launch_bounds__(kThreads) std_normal_log_prob_kernel(const float* __restrict__ z, int64_t ldz, int d,
                                                                       float log_z, const float* __restrict__ lad,
                                                                       float* __restrict__ out, int64_t n_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp0; r < n_rows; r += n_warps) {
        const float* zr = z + r * ldz;
        float acc = 0.0f;
        if ((d & 3) == 0 && (ldz & 3) == 0 && (reinterpret_cast<uintptr_t>(z) & 15u) == 0) {
            const float4* z4 = reinterpret_cast<const float4*>(zr);
            for (int j = lane; j < (d >> 2); j += 32) {
                float4 v = __ldcs(z4 + j);
                acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
            }
        } else {
            for (int j = lane; j < d; j += 32) { float v = zr[j]; acc += v * v; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) {
            float lp = -0.5f * acc - log_z;
            out[r] = lad ? lp + lad[r] : lp;
        }
    }
}

}  // namespace nfk

using namespace nfk;

extern "C" int nfk_gather_cols(const float* x, int64_t ldx, const int32_t* cols, int32_t n_cols, float* out, int64_t ldo,
                               int64_t n_rows, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && n_cols >= 0, "bad sizes");
    if (n_rows == 0 || n_cols == 0) return NFK_OK;
    NFK_REQUIRE(x && cols && out, "NULL pointer");
    gather_cols_kernel<<<grid_for(n_rows * n_cols, kThreads), kThreads, 0, (cudaStream_t)stream>>>(x, ldx, cols, n_cols, out,
                                                                                                    ldo, n_rows);
    return check_launch("gather_cols_kernel");
}

extern "C" int nfk_actnorm(const float* x, int64_t ldx, const float* scale, const float* shift, float* y, int64_t ldy,
                           float* lad_accum, float lad_const, int64_t n_rows, int32_t d, int inverse, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && d >= 1, "bad sizes");
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(x && scale && shift && y, "NULL pointer");
    actnorm_kernel<<<grid_for(n_rows * d, kThreads), kThreads, 0, (cudaStream_t)stream>>>(x, ldx, scale, shift, y, ldy,
                                                                                          lad_accum, lad_const, n_rows, d,
                                                                                          inverse);
    return check_launch("actnorm_kernel");
}

extern "C" int nfk_add_const(float* lad_accum, float c, int64_t n_rows, void* stream) {
    NFK_REQUIRE(n_rows >= 0, "bad size");
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(lad_accum, "NULL pointer");
    add_const_kernel<<<grid_for(n_rows, kThreads), kThreads, 0, (cudaStream_t)stream>>>(lad_accum, c, n_rows);
    return check_launch("add_const_kernel");
}

// max |x| of a (possibly strided) matrix into *out (a non-negative float, so its bit pattern orders like an int):
// *out must hold 0.0f on entry.  NaNs are skipped (fmaxf).
__global__ void absmax_kernel(const float* __restrict__ x, int64_t ldx, int64_t n_rows, int n_cols, float* out) {
    float m = 0.0f;
    const int64_t total = n_rows * n_cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / n_cols;
        m = fmaxf(m, fabsf(x[r * ldx + (i - r * n_cols)]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    // one atomic per block, not per warp: the gradient exponents of a training step read this for every layer
    __shared__ float warp_max[kThreads / 32];
    if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kThreads / 32; ++w) m = fmaxf(m, warp_max[w]);
        if (m > 0.0f) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));
    }
}

extern "C" int nfk_absmax(const float* x, int64_t ldx, int64_t n_rows, int32_t n_cols, float* out, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && n_cols >= 0, "bad sizes");
    NFK_REQUIRE(out, "NULL pointer");
    if (n_rows == 0 || n_cols == 0) return NFK_OK;
    NFK_REQUIRE(x, "NULL pointer");
    absmax_kernel<<<grid_for(n_rows * n_cols, kThreads), kThreads, 0, (cudaStream_t)stream>>>(x, ldx, n_rows, n_cols, out);
    return check_launch("absmax_kernel");
}

extern "C" int nfk_fill(float* dst, float value, int64_t n, void* stream) {
    NFK_REQUIRE(n >= 0, "bad size");
    if (n == 0) return NFK_OK;
    NFK_REQUIRE(dst, "NULL pointer");
    fill_kernel<<<grid_for(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(dst, value, n);
    return check_launch("fill_kernel");
}

extern "C" int nfk_affine_coupling_rows(const float* x, int64_t ldx, const float* params, int32_t mult,
                                        int32_t scale_activation, int inverse, const int32_t* t_cols, int32_t d_t,
                                        const int32_t* id_cols, int32_t d_id, float* y, int64_t ldy, float* lad_accum,
                                        int64_t n_rows, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && d_t >= 1 && d_id >= 0, "bad sizes");
    NFK_REQUIRE(mult == 1 || mult == 2, "mult must be 1 (additive) or 2 (affine)");
    NFK_REQUIRE(scale_activation == 0 || scale_activation == 1, "unknown scale activation %d", scale_activation);
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(x && params && y, "NULL pointer");
    NFK_REQUIRE(d_id == 0 || id_cols, "id_cols is NULL");
    NFK_REQUIRE(x != y, "y must not alias x");
    affine_coupling_rows_kernel<<<grid_for(n_rows * 32, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
        x, ldx, params, mult, scale_activation, inverse, t_cols, d_t, id_cols, d_id, y, ldy, lad_accum, n_rows);
    return check_launch("affine_coupling_rows_kernel");
}

extern "C" int nfk_std_normal_log_prob(const float* z, int64_t ldz, int32_t d, float log_z, const float* lad, float* out,
                                       int64_t n_rows, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && d >= 1, "bad sizes");
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(z && out, "NULL pointer");
    std_normal_log_prob_kernel<<<grid_for(n_rows * 32, kThreads), kThreads, 0, (cudaStream_t)stream>>>(z, ldz, d, log_z, lad,
                                                                                                       out, n_rows);
    return check_launch("std_normal_log_prob_kernel");
}
