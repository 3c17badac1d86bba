// Rational-quadratic spline kernels (HBM-bound): the functional elementwise API and the coupling epilogue that
// consumes conditioner outputs stored in HBM.  See include/nfk.h for the reference lines each one replaces.
#include <math.h>

#include <algorithm>

#include "nfk_common.cuh"
#include "rq_spline.cuh"

namespace nfk {

int make_spline_params(const NfkSplineDesc* d, SplineParams* p) {
    if (!d) return fail(NFK_E_INVALID, "spline desc is NULL");
    const int K = d->num_bins;
    if (K < 1 || K > NFK_MAX_BINS) return fail(NFK_E_INVALID, "num_bins=%d outside [1,%d]", K, NFK_MAX_BINS);
    // reference raises ValueError for these (rational_quadratic.py:86-89); the host mirror raises before calling.
    if (d->min_bin_width * K > 1.0) return fail(NFK_E_INVALID, "Minimal bin width too large for the number of bins");
    if (d->min_bin_height * K > 1.0) return fail(NFK_E_INVALID, "Minimal bin height too large for the number of bins");
    *p = spline_params_of(*d);
    return NFK_OK;
}

// ------------------------------------------------------------------------------------------------------------
// elementwise API: one thread per element, parameters read straight from global memory
// ------------------------------------------------------------------------------------------------------------
template <int KMAX, bool EXACT>
__global__ void __launch_bounds__(256) rqs_elementwise_kernel(SplineParams p, int inverse, const float* __restrict__ x,
                                                              const float* __restrict__ uw, const float* __restrict__ uh,
                                                              const float* __restrict__ ud, int64_t stride_w,
                                                              int64_t stride_h, int64_t stride_d, int64_t period,
                                                              float* __restrict__ y, float* __restrict__ lad,
                                                              int64_t n_elem, int32_t* flags) {
    int flag = 0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_elem; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = period > 0 ? e % period : e;
        float w[KMAX], h[KMAX], d[KMAX + 1];
        const float* pw = uw + r * stride_w;
        const float* ph = uh + r * stride_h;
        const float* pd = ud + r * stride_d;
        rqs_load<KMAX, EXACT>(p, [&](int k) { return __ldg(pw + k); }, [&](int k) { return __ldg(ph + k); },
                              [&](int k) { return __ldg(pd + k); }, w, h, d);
        float yy, ll;
        rqs_eval<KMAX, EXACT>(p, inverse != 0, x[e], w, h, d, yy, ll, flag);
        y[e] = yy;
        lad[e] = ll;
    }
    if (flag && flags) atomicOr(flags, flag);
}

// ------------------------------------------------------------------------------------------------------------
// coupling epilogue: params [n_rows, d_t*M] in HBM, staged through shared memory in 128-element chunks
// ------------------------------------------------------------------------------------------------------------
constexpr int kRowsThreads = 128;

// One block = 128 threads = 128 consecutive (row, feature) elements per chunk.  The parameters of a chunk are one
// contiguous run of 128*M floats: they are fetched with coalesced 16-byte loads into REGISTERS one chunk ahead (so the
// HBM latency of chunk c+1 is covered by the arithmetic of chunk c), parked in shared memory, and read back one element per
// thread (stride M words: conflict-free for odd M).
template <int KMAX, bool EXACT>
__global__ void __launch_bounds__(kRowsThreads) rqs_rows_kernel(SplineParams p, int inverse, const float* __restrict__ x,
                                                                int64_t ldx, const float* __restrict__ params,
                                                                const int32_t* __restrict__ t_cols, int d_t,
                                                                const int32_t* __restrict__ id_cols, int d_id,
                                                                float* __restrict__ y, int64_t ldy,
                                                                float* __restrict__ lad_accum, int64_t n_rows,
                                                                int rows_per_group, int32_t* flags) {
    extern __shared__ __align__(16) float sp[];   // [kRowsThreads * M] staged parameters, then [kRowsThreads] lad
    // float4 per thread staged in registers = ceil(M_max / 4); register prefetch only for the common small bin counts
    constexpr int kMaxPrefetch = KMAX <= 16 ? (spline_param_count(KMAX, false) + 3) / 4 : 1;
    const int M = spline_param_count(EXACT ? KMAX : p.num_bins, p.linear_tails);
    float* s_lad = sp + kRowsThreads * M;
    const int tid = threadIdx.x;
    const int64_t n_groups = (n_rows + rows_per_group - 1) / rows_per_group;
    const bool pow2_rows = rows_per_group > 1 && (d_t & (d_t - 1)) == 0 && d_t <= 32;   // a row = an aligned lane group
    const bool use_prefetch = KMAX <= 16 && (kRowsThreads * M + 3) / 4 <= kMaxPrefetch * kRowsThreads;
    int flag = 0;
    // element index -> (row in group, feature): shifts when the feature counts are powers of two (integer division is ~20
    // instructions, and this kernel is issue-bound: ncu r2, 71 % issue-slot utilisation at 48 % of DRAM bandwidth)
    const int sh_t = (d_t & (d_t - 1)) == 0 ? 31 - __clz(d_t) : -1;
    const int sh_id = (d_id > 0 && (d_id & (d_id - 1)) == 0) ? 31 - __clz(d_id) : -1;

    float4 pre[kMaxPrefetch];
    // chunk (g, e0): elements [e0, e0 + cnt) of row group g
    auto chunk_src = [&](int64_t g, int e0) { return params + ((g * rows_per_group) * d_t + e0) * (int64_t)M; };
    auto chunk_cnt = [&](int64_t g, int e0) {
        const int rows_here = (int)min((int64_t)rows_per_group, n_rows - g * rows_per_group);
        return min(kRowsThreads, rows_here * d_t - e0);
    };
    auto prefetch = [&](const float* src, int n_f) {
        const float4* src4 = reinterpret_cast<const float4*>(src);
#pragma unroll
        for (int u = 0; u < kMaxPrefetch; ++u) {
            const int i = tid + u * kRowsThreads;
            if (i < (n_f >> 2)) pre[u] = __ldcs(src4 + i);
        }
    };
    auto park = [&](const float* src, int n_f, bool fetched) {
        if (fetched) {
            float4* dst4 = reinterpret_cast<float4*>(sp);
#pragma unroll
            for (int u = 0; u < kMaxPrefetch; ++u) {
                const int i = tid + u * kRowsThreads;
                if (i < (n_f >> 2)) dst4[i] = pre[u];
            }
            for (int i = (n_f & ~3) + tid; i < n_f; i += kRowsThreads) sp[i] = __ldcs(src + i);
        } else {
            for (int i = tid; i < n_f; i += kRowsThreads) sp[i] = __ldcs(src + i);
        }
    };

    int64_t g = blockIdx.x;
    int e0 = 0;
    bool have = false;               // registers hold the chunk (g, e0)
    if (g < n_groups) {
        const float* src = chunk_src(g, e0);
        have = use_prefetch && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0);
        if (have) prefetch(src, chunk_cnt(g, e0) * M);
    }
    float my_lad = 0.0f;
    while (g < n_groups) {
        const int64_t row0 = g * rows_per_group;
        const int rows_here = (int)min((int64_t)rows_per_group, n_rows - row0);
        const int n_el = rows_here * d_t;
        const int cnt = min(kRowsThreads, n_el - e0);
        park(chunk_src(g, e0), cnt * M, have);
        __syncthreads();
        // next chunk: same group if it has more elements, else the next group of this block
        int64_t ng = g;
        int ne0 = e0 + kRowsThreads;
        if (ne0 >= n_el) { ng = g + gridDim.x; ne0 = 0; }
        have = false;
        if (ng < n_groups) {
            const float* nsrc = chunk_src(ng, ne0);
            have = use_prefetch && ((reinterpret_cast<uintptr_t>(nsrc) & 15u) == 0);
            if (have) prefetch(nsrc, chunk_cnt(ng, ne0) * M);
        }

        float ll = 0.0f;
        if (tid < cnt) {
            const int e = e0 + tid;
            const int r = sh_t >= 0 ? e >> sh_t : e / d_t;
            const int j = e - r * d_t;
            const int col = t_cols ? __ldg(t_cols + j) : j;
            const int64_t row = row0 + r;
            const float* q = sp + tid * M;
            auto at = [&](int i) { return q[i]; };
            float yy;
            if (EXACT) {
                // compile-time bin count: the lean form (binary bin search, template direction) straight on the staged parameters
                rqs_eval_lean_one<KMAX>(p, inverse, x[row * ldx + col], at, yy, ll, flag);
            } else {
                float w[KMAX], h[KMAX], d[KMAX + 1];
                rqs_load_packed<KMAX, EXACT>(p, at, w, h, d);
                rqs_eval<KMAX, EXACT>(p, inverse != 0, x[row * ldx + col], w, h, d, yy, ll, flag);
            }
            y[row * ldy + col] = yy;
        }

        if (rows_per_group == 1) {
            my_lad += ll;
        } else if (pow2_rows) {
            // a row is d_t consecutive lanes inside one warp: butterfly over the lane group, fixed order
            float v = ll;
            for (int o = d_t >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lad_accum && tid < cnt && (tid & (d_t - 1)) == 0) lad_accum[row0 + tid / d_t] += v;
        } else {
            s_lad[tid] = ll;
        }
        __syncthreads();

        const bool group_done = (ne0 == 0);
        if (group_done) {
            // identity columns: bit-exact copy (coupling.py:96-97)
            for (int e = tid; e < rows_here * d_id; e += kRowsThreads) {
                const int r = sh_id >= 0 ? e >> sh_id : e / d_id;
                const int col = __ldg(id_cols + (e - r * d_id));
                y[(row0 + r) * ldy + col] = __ldcs(x + (row0 + r) * ldx + col);
            }
            if (lad_accum) {
                if (rows_per_group == 1) {
                    block_sum_in_order(my_lad, s_lad, kRowsThreads / 32, [&](float t) { lad_accum[row0] += t; });
                    my_lad = 0.0f;
                } else if (!pow2_rows) {
                    // single chunk by construction (rows_per_group * d_t <= kRowsThreads): fixed-order per-row sums
                    if (tid < rows_here) {
                        float t = 0.0f;
                        for (int j = 0; j < d_t; ++j) t += s_lad[tid * d_t + j];
                        lad_accum[row0 + tid] += t;
                    }
                    __syncthreads();
                }
            }
        }
        g = ng;
        e0 = ne0;
    }
    if (flag && flags) atomicOr(flags, flag);
}

template <int KMAX, bool EXACT>
static int launch_rows(const SplineParams& p, int inverse, const float* x, int64_t ldx, const float* params,
                       const int32_t* t_cols, int d_t, const int32_t* id_cols, int d_id, float* y, int64_t ldy,
                       float* lad_accum, int64_t n_rows, int32_t* flags, cudaStream_t st) {
    const int M = spline_param_count(p.num_bins, p.linear_tails);
    const size_t smem = (size_t)(kRowsThreads * M + kRowsThreads) * sizeof(float);
    if (int rc = allow_dynamic_smem(rqs_rows_kernel<KMAX, EXACT>, smem)) return rc;
    const int rpg = d_t >= kRowsThreads ? 1 : max(1, kRowsThreads / d_t);
    const int64_t n_groups = (n_rows + rpg - 1) / rpg;
    const int grid = (int)std::min<int64_t>(n_groups, (int64_t)tc::sm_count() * 32);
    rqs_rows_kernel<KMAX, EXACT><<<grid, kRowsThreads, smem, st>>>(p, inverse, x, ldx, params, t_cols, d_t, id_cols, d_id, y, ldy,
                                                            lad_accum, n_rows, rpg, flags);
    return check_launch("rqs_rows_kernel");
}

}  // namespace nfk

using namespace nfk;

extern "C" int nfk_rqs_elementwise(const NfkSplineDesc* desc, int inverse, const float* x, const float* uw,
                                   const float* uh, const float* ud, int64_t stride_w, int64_t stride_h,
                                   int64_t stride_d, int64_t param_period, float* y, float* lad, int64_t n_elem,
                                   int32_t* flags, void* stream) {
    SplineParams p;
    int rc = make_spline_params(desc, &p);
    if (rc) return rc;
    NFK_REQUIRE(n_elem >= 0, "n_elem < 0");
    if (n_elem == 0) return NFK_OK;
    // one bin with linear tails has no interior derivative (K - 1 = 0): an empty ud, whose pointer may be NULL, is never read
    const bool needs_ud = !(p.linear_tails && p.num_bins == 1);
    NFK_REQUIRE(x && uw && uh && (ud || !needs_ud) && y && lad, "NULL tensor pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int threads = 256;
    const int grid = (int)std::min<int64_t>((n_elem + threads - 1) / threads, (int64_t)tc::sm_count() * 64);
    with_bin_instance(p.num_bins, [&](auto km, auto ex) {
        rqs_elementwise_kernel<km, ex><<<grid, threads, 0, st>>>(p, inverse, x, uw, uh, ud, stride_w, stride_h, stride_d,
                                                                 param_period, y, lad, n_elem, flags);
    });
    return check_launch("rqs_elementwise_kernel");
}

extern "C" int nfk_rqs_rows(const NfkSplineDesc* desc, int inverse, const float* x, int64_t ldx, const float* params,
                            const int32_t* t_cols, int32_t d_t, const int32_t* id_cols, int32_t d_id, float* y,
                            int64_t ldy, float* lad_accum, int64_t n_rows, int32_t* flags, void* stream) {
    SplineParams p;
    int rc = make_spline_params(desc, &p);
    if (rc) return rc;
    NFK_REQUIRE(n_rows >= 0 && d_t >= 1 && d_id >= 0, "bad sizes n_rows=%lld d_t=%d d_id=%d", (long long)n_rows, d_t, d_id);
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(x && params && y, "NULL tensor pointer");
    NFK_REQUIRE(d_id == 0 || id_cols, "id_cols is NULL");
    NFK_REQUIRE(x != y, "y must not alias x");
    cudaStream_t st = (cudaStream_t)stream;
    return with_bin_instance(p.num_bins, [&](auto km, auto ex) {
        return launch_rows<km, ex>(p, inverse, x, ldx, params, t_cols, d_t, id_cols, d_id, y, ldy, lad_accum, n_rows, flags, st);
    });
}
