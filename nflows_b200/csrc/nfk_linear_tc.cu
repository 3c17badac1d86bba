// Dense layer on the Hopper tensor cores (wgmma) with fp32-equivalent operand precision.
//
//   Y = post(A W^T + b) + R           A: [n_rows, K]   W: [N, K] (nn.Linear layout)   fp32 accumulate
//
// PyTorch's reference GEMM is true fp32 (allow_tf32=False); one reduced-precision pass misses the 1e-5 parity bar by two
// orders of magnitude (SURVEY.md Appendix C).  So every operand is carried as a split pair of fp16 numbers
//   v * 2^e = v_hi + v_lo,   v_hi = rn_fp16(v * 2^e),   v_lo = rn_fp16(v * 2^e - v_hi)        (22 mantissa bits)
// with a per-tensor power-of-two scale 2^e that keeps v_lo out of the fp16 subnormals (weights: max |w| -> 2^14;
// activations: a fixed exponent, overflow raises NFK_FLAG_F16_RANGE), and each K-step issues three f16 MMAs into the
// same accumulator:  a_lo*w_hi + a_hi*w_lo + a_hi*w_hi  (the dropped a_lo*w_lo term is ~2^-22 relative; fp16 x fp16
// products are exact in the fp32 accumulator).  The epilogue multiplies by 2^-(e_a + e_w), exactly.  fp16 pairs carry the
// same 22 bits as a 3xTF32 scheme at half the operand bytes and twice the K per MMA instruction.
//
// Accumulation: the tensor core adds into its fp32 accumulator with round-toward-zero, so a long chain of MMAs acquires
// a bias of ~0.5 ulp per instruction (the effect Ootomo & Yokota 2022 report for Ampere).  The accumulator therefore only
// ever holds a PARTIAL sum over DRAIN_SLABS_LINEAR K-slabs (12 MMAs), which is added to running sums in registers with
// round-to-nearest FADDs (tc_common.cuh: mma_tile).
//
// Kernel shape (tc_common.cuh): one persistent CTA per SM, a TMA producer warpgroup and two consumer warpgroups of 64 rows
// each; tiles of 128 rows x 128 columns, numbered column tile fastest and handed out to the CTAs in that order, so that the
// column tiles of a row block run at the same time on neighbouring CTAs and its A slabs come from HBM once, then from L2.  The epilogue works on the accumulator fragments in registers: bias (and a residual
// that no relu separates from the sum) start the running sums, the finished values are stored straight from registers
// (fp32 result and / or the fp16 pair the next layer multiplies), or -- affine coupling -- consumed as (shift, scale) pairs.
#include <stdlib.h>

#include <mutex>

#include "tc_common.cuh"

namespace nfk {
namespace tc {

struct Params {
    const float* bias;       // [N] or null
    const float* residual;   // [n_rows, ldr] or null
    float* y;                // fp32 result or null
    __half* y_hi;            // fp16 split pair of pre(y) * out_scale for the next layer, or null
    __half* y_lo;
    int32_t* flags;          // NFK_FLAG_F16_RANGE when a pair output leaves the fp16 range
    float acc_scale;         // 2^(e_a + e_w): the accumulators hold (A W^T) * acc_scale
    float inv_acc_scale;
    float out_scale;         // 2^e of the pair output
    int split_n;             // pair output for columns < split_n only
    int64_t ldr, ldy, lds;
    int64_t n_rows;
    int K, N;
    int relu_out;            // relu applied to (acc + bias) before the residual add / store
    int split_relu;          // relu applied before splitting (the next layer consumes relu(y))
    int num_m_tiles, num_n_tiles;
    int y_first_col;         // the fp32 result is only needed for columns >= y_first_col
    int drain;               // K-slabs accumulated by the tensor core per partial sum (DRAIN_SLABS_LINEAR)
    // affine-coupling epilogue (nfk_affine_coupling_final_f16x3): the GEMM result is the conditioner's parameter row --
    // interleaved (shift_j, raw scale_j) pairs when c_mult == 2, shift_j when 1 -- consumed in registers, never stored
    const float* cx;         // coupling input [n_rows, ldcx]; NULL = plain dense layer
    float* cy;               // coupling output [n_rows, ldcy] (transformed columns only; may alias cx)
    const int32_t* c_cols;   // column of transformed feature j, or NULL: c_col0 + j
    float* c_lad;            // running log|det| per row (atomicAdd of this thread's share), may be NULL
    int64_t ldcx, ldcy;
    int c_col0, c_dt, c_mult, c_act, c_inverse;
};

constexpr int LIN_STAGES = 6;                                           // 6 x 32 KB ring
constexpr int LIN_SMEM_BYTES = LIN_STAGES * STAGE_BYTES + 256 /*barriers*/ + 1024 /*alignment slack*/;

// ACT: the instance for activation codes other than none and relu; the other applies relu only, as it always did.
template <bool ACT>
__device__ __forceinline__ float act_of(int code, float x) {
    if constexpr (ACT) return nfk_act(code, x);
    return fmaxf(x, 0.0f);
}

template <bool ACT>
__global__ void __launch_bounds__(THREADS, 1)
linear_f16x3_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                    const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo, const Params p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;      // swizzle atoms need (at least) 512-byte alignment
    const uint32_t bars = smem_base + LIN_STAGES * STAGE_BYTES;
    Ring ring{smem_base, bars, bars + 8 * LIN_STAGES, LIN_STAGES, (uint32_t)STAGE_BYTES};
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_k = (p.K + BK - 1) / BK;
    const int num_tiles = p.num_m_tiles * p.num_n_tiles;

    if (threadIdx.x == 0) {
        for (int s = 0; s < LIN_STAGES; ++s) { mbar_init(ring.full + 8 * s, 1); mbar_init(ring.empty + 8 * s, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        prefetch_tmap(&map_a_hi); prefetch_tmap(&map_a_lo); prefetch_tmap(&map_w_hi); prefetch_tmap(&map_w_lo);
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");      // registers to the consumer warpgroups
        // ================================================= TMA producer (one elected thread of warp 0)
        if (warp == 0 && elect_one()) {
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const int m0 = (t / p.num_n_tiles) * BM, n0 = (t % p.num_n_tiles) * BN;
                for (int ks = 0; ks < num_k; ++ks) produce_slab(ring, &map_a_hi, &map_a_lo, &map_w_hi, &map_w_lo, ks, m0, n0);
            }
        }
        return;
    }
    // ================================================= consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int wg = (warp >> 2) - 1, wi = warp & 3;
    const int q = lane & 3;
    int flag = 0;
    const bool fold_residual = p.residual && !p.relu_out;
    const bool vec_y = p.y && (p.ldy % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.y) & 7) == 0);
    const bool vec_s = p.y_hi && (p.lds % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.y_hi) & 3) == 0) &&
                       ((reinterpret_cast<uintptr_t>(p.y_lo) & 3) == 0);
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int tm = t / p.num_n_tiles, tn = t % p.num_n_tiles;
        int64_t rows[2];
        rows[0] = (int64_t)tm * BM + wg * 64 + wi * 16 + (lane >> 2);
        rows[1] = rows[0] + 8;
        const int c_base = tn * BN + 2 * q;                   // column of sum[4 j + (i & 1)] is c_base + 8 j + (i & 1)
        // running sums start from the bias (+ a residual no relu separates from the sum), in the accumulators' power-of-two
        // scaled domain (exact)
        float sum[64];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = c_base + 8 * j + e;
                const float b = (p.bias && col < p.N) ? __ldg(p.bias + col) * p.acc_scale : 0.0f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float r = 0.0f;
                    if (fold_residual && col < p.N && rows[h] < p.n_rows) r = p.residual[rows[h] * p.ldr + col];
                    sum[4 * j + 2 * h + e] = fmaf(r, p.acc_scale, b);
                }
            }
        }
        mma_tile(sum, ring, num_k, p.drain, wg, lane);
        if (p.cx) {
            // ---- affine / additive coupling (coupling.py:212-269 of the reference) on the parameters held in registers:
            // y_j = x_j * s_j + t_j (inverse: (x_j - t_j) / s_j), log|det| += +-sum_j log s_j
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = rows[h];
                if (row >= p.n_rows) continue;
                float lad = 0.0f;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = c_base + 8 * j;                // even
                    if (col >= p.N) continue;
                    const float a0 = sum[4 * j + 2 * h] * p.inv_acc_scale, a1 = sum[4 * j + 2 * h + 1] * p.inv_acc_scale;
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int jf = p.c_mult == 2 ? (col >> 1) : col + e;
                        if ((p.c_mult == 2 && e == 1) || jf >= p.c_dt) continue;
                        const int cf = p.c_cols ? __ldg(p.c_cols + jf) : p.c_col0 + jf;
                        const float x = p.cx[row * p.ldcx + cf];
                        const float shift = (p.c_mult == 2 || e == 0) ? a0 : a1;
                        float out;
                        if (p.c_mult == 2) {
                            float scale;
                            if (p.c_act == 0) {
                                scale = 1.0f / (1.0f + expf(-(a1 + 2.0f))) + 1e-3f;
                            } else {
                                const float sp = a1 > 20.0f ? a1 : log1pf(expf(a1));
                                scale = fminf(fmaxf(sp + 1e-3f, 0.0f), 3.0f);
                            }
                            lad += logf(scale);
                            out = p.c_inverse ? __fdiv_rn(__fsub_rn(x, shift), scale) : __fadd_rn(__fmul_rn(x, scale), shift);
                        } else {
                            out = p.c_inverse ? (x - shift) : (x + shift);
                        }
                        p.cy[row * p.ldcy + cf] = out;
                    }
                }
                if (p.c_lad && p.c_mult == 2) atomicAdd(p.c_lad + row, p.c_inverse ? -lad : lad);
            }
            continue;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = rows[h];
            if (row >= p.n_rows) continue;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = c_base + 8 * j;
                if (col >= p.N) continue;
                const bool two = col + 1 < p.N;
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float x = sum[4 * j + 2 * h + e] * p.inv_acc_scale;       // bias (and a foldable residual) already included
                    if (p.relu_out) x = act_of<ACT>(p.relu_out, x);
                    if (p.residual && !fold_residual && (e == 0 || two)) x += p.residual[row * p.ldr + col + e];
                    v[e] = x;
                }
                if (p.y && col + 2 > p.y_first_col) {
                    float* yp = p.y + row * p.ldy + col;
                    if (vec_y && two && col >= p.y_first_col) {
                        *reinterpret_cast<float2*>(yp) = make_float2(v[0], v[1]);
                    } else {
                        if (col >= p.y_first_col) yp[0] = v[0];
                        if (two) yp[1] = v[1];
                    }
                }
                if (p.y_hi && col < p.split_n) {
                    __half hi[2], lo[2];
                    const int n_out = (two && col + 1 < p.split_n) ? 2 : 1;
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        if (e < n_out) split_f16(p.split_relu ? act_of<ACT>(p.split_relu, v[e]) : v[e], p.out_scale, hi[e], lo[e], flag);
                    __half* hp = p.y_hi + row * p.lds + col;
                    __half* lp = p.y_lo + row * p.lds + col;
                    if (vec_s && n_out == 2) {
                        *reinterpret_cast<__half2*>(hp) = __halves2half2(hi[0], hi[1]);
                        *reinterpret_cast<__half2*>(lp) = __halves2half2(lo[0], lo[1]);
                    } else {
                        hp[0] = hi[0]; lp[0] = lo[0];
                        if (n_out == 2) { hp[1] = hi[1]; lp[1] = lo[1]; }
                    }
                }
            }
        }
    }
    if (flag && p.flags) atomicOr(p.flags, flag);
}

// ---------------------------------------------------------------- fp32 -> fp16 (hi, lo) split pair, optional activation
// HBM-bound: 4 B read + 4 B written per element.  Used for weights (once per parameter update), for tensors entering a
// tensor-core chain from outside and for the transformed half of a coupling output.
__global__ void __launch_bounds__(256) split_f16_kernel(const float* __restrict__ x, int64_t ldx, int n_cols, int relu,
                                                        float scale, __half* __restrict__ hi, __half* __restrict__ lo,
                                                        int64_t ldo, int64_t n_rows, int vec4, int32_t* flags) {
    int flag = 0;
    if (vec4) {
        const int n4 = n_cols >> 2;
        const int64_t total = n_rows * n4;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
            const int64_t r = i / n4;
            const int j = (int)(i - r * n4) * 4;
            float4 v = __ldcs(reinterpret_cast<const float4*>(x + r * ldx + j));
            if (relu == NFK_ACT_RELU) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            else if (relu) { v.x = nfk_act(relu, v.x); v.y = nfk_act(relu, v.y); v.z = nfk_act(relu, v.z); v.w = nfk_act(relu, v.w); }
            __half h[4], l[4];
            split_f16(v.x, scale, h[0], l[0], flag); split_f16(v.y, scale, h[1], l[1], flag);
            split_f16(v.z, scale, h[2], l[2], flag); split_f16(v.w, scale, h[3], l[3], flag);
            *reinterpret_cast<uint2*>(hi + r * ldo + j) = *reinterpret_cast<const uint2*>(h);
            *reinterpret_cast<uint2*>(lo + r * ldo + j) = *reinterpret_cast<const uint2*>(l);
        }
    } else {
        const int64_t total = n_rows * n_cols;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
            const int64_t r = i / n_cols;
            const int j = (int)(i - r * n_cols);
            float v = x[r * ldx + j];
            if (relu) v = nfk_act(relu, v);
            __half h, l;
            split_f16(v, scale, h, l, flag);
            hi[r * ldo + j] = h;
            lo[r * ldo + j] = l;
        }
    }
    if (flag && flags) atomicOr(flags, flag);
}

// Context gate of a residual block (nn/nets/resnet.py:50-53): y = skip + t * sigmoid(gate), i.e. F.glu(cat(t, gate)) + inputs,
// in one pass; writes the fp32 result (the next block's skip tensor) and/or the fp16 pair the next dense layer multiplies.
__global__ void __launch_bounds__(256) glu_skip_kernel(const float* __restrict__ t, int64_t ldt, const float* __restrict__ gate,
                                                       int64_t ldg, const float* __restrict__ skip, int64_t ldsk, float* __restrict__ y,
                                                       int64_t ldy, __half* __restrict__ hi, __half* __restrict__ lo, int64_t ldo,
                                                       float scale, int relu, int64_t n_rows, int n_cols, int32_t* flags) {
    int flag = 0;
    const int64_t total = n_rows * n_cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / n_cols;
        const int j = (int)(i - r * n_cols);
        const float g = gate[r * ldg + j];
        float v = t[r * ldt + j] * (1.0f / (1.0f + expf(-g)));
        if (skip) v += skip[r * ldsk + j];
        if (y) y[r * ldy + j] = v;
        if (hi) {
            __half h, l;
            split_f16(relu ? nfk_act(relu, v) : v, scale, h, l, flag);
            hi[r * ldo + j] = h;
            lo[r * ldo + j] = l;
        }
    }
    if (flag && flags) atomicOr(flags, flag);
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(sym);
    });
    return fn;
}

// K-major fp16 operand: boxes of {BK, box_rows}, SWIZZLE_64B, out-of-bounds elements read as zero
int make_map(CUtensorMap* map, const __half* base, int64_t rows, int K, int64_t ld, int box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return fail(NFK_E_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(NFK_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return NFK_OK;
}

int sm_count() {
    static std::atomic<int> counts[64];                      // per device
    int dev = 0;
    cudaGetDevice(&dev);
    int n = counts[dev & 63].load(std::memory_order_relaxed);
    if (!n) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
        counts[dev & 63].store(n, std::memory_order_relaxed);
    }
    return n;
}

}  // namespace tc
}  // namespace nfk

using namespace nfk;

static bool pow2_exp_ok(int e) { return e >= -60 && e <= 60; }

extern "C" int nfk_split_f16(const float* x, int64_t ldx, int32_t n_cols, int relu, int32_t scale_exp, void* hi, void* lo,
                             int64_t ldo, int64_t n_rows, int32_t* flags, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && n_cols >= 0 && pow2_exp_ok(scale_exp), "bad sizes");
    NFK_REQUIRE(act_valid(relu), "unknown activation code (relu=%d)", relu);
    if (n_rows == 0 || n_cols == 0) return NFK_OK;
    NFK_REQUIRE(x && hi && lo, "NULL pointer");
    const int vec4 = (n_cols % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0 && aligned16(x) && (reinterpret_cast<uintptr_t>(hi) & 7) == 0 &&
                      (reinterpret_cast<uintptr_t>(lo) & 7) == 0) ? 1 : 0;
    int64_t blocks = (n_rows * (vec4 ? n_cols / 4 : n_cols) + 255) / 256;
    const int64_t cap = (int64_t)tc::sm_count() * 32;
    int grid = (int)(blocks > cap ? cap : blocks);
    tc::split_f16_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, n_cols, relu, ldexpf(1.0f, scale_exp), (__half*)hi, (__half*)lo,
                                                                 ldo, n_rows, vec4, flags);
    return check_launch("split_f16_kernel");
}

extern "C" int nfk_glu_skip_rows(const float* t, int64_t ldt, const float* gate, int64_t ldg, const float* skip, int64_t ldsk,
                                 float* y, int64_t ldy, void* y_hi, void* y_lo, int64_t lds, int32_t y_exp, int split_relu,
                                 int64_t n_rows, int32_t n_cols, int32_t* flags, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && n_cols >= 0 && pow2_exp_ok(y_exp), "bad sizes");
    NFK_REQUIRE(act_valid(split_relu), "unknown activation code (split_relu=%d)", split_relu);
    if (n_rows == 0 || n_cols == 0) return NFK_OK;
    NFK_REQUIRE(t && gate, "NULL pointer");
    NFK_REQUIRE(y || (y_hi && y_lo), "no output requested");
    NFK_REQUIRE((y_hi == nullptr) == (y_lo == nullptr), "y_hi and y_lo must be given together");
    int64_t blocks = (n_rows * n_cols + 255) / 256;
    const int64_t cap = (int64_t)tc::sm_count() * 32;
    int grid = (int)(blocks > cap ? cap : blocks);
    tc::glu_skip_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(t, ldt, gate, ldg, skip, ldsk, y, ldy, (__half*)y_hi, (__half*)y_lo, lds,
                                                                ldexpf(1.0f, y_exp), split_relu, n_rows, n_cols, flags);
    return check_launch("glu_skip_kernel");
}

// fp16 rows must start on 16-byte boundaries for TMA: leading dimensions and K multiples of 8
extern "C" int nfk_linear_f16x3_supported(int64_t lda, int64_t ldw, int32_t in_features) {
    return (in_features >= 8 && in_features % 8 == 0 && lda % 8 == 0 && ldw % 8 == 0) ? 1 : 0;
}

namespace {
struct CouplingEpilogue {        // set by nfk_affine_coupling_final_f16x3
    const float* x; int64_t ldx; float* y; int64_t ldy; const int32_t* t_cols; int t_col0, d_t, mult, act, inverse; float* lad;
};
}  // namespace

static int linear_f16x3_launch(const void* a_hi_, const void* a_lo_, int64_t lda, int32_t a_exp, const void* w_hi_,
                               const void* w_lo_, int64_t ldw, int32_t w_exp, const float* bias, const float* R, int64_t ldr,
                               float* Y, int64_t ldy, void* y_hi_, void* y_lo_, int64_t lds, int32_t y_exp, int32_t split_cols,
                               int32_t y_first_col, int relu_out, int split_relu, int64_t n_rows, int32_t in_features,
                               int32_t out_features, int32_t* flags, void* stream, const CouplingEpilogue* ce);

extern "C" int nfk_linear_f16x3(const void* a_hi_, const void* a_lo_, int64_t lda, int32_t a_exp, const void* w_hi_,
                                const void* w_lo_, int64_t ldw, int32_t w_exp, const float* bias, const float* R, int64_t ldr,
                                float* Y, int64_t ldy, void* y_hi_, void* y_lo_, int64_t lds, int32_t y_exp, int32_t split_cols,
                                int32_t y_first_col, int relu_out, int split_relu, int64_t n_rows, int32_t in_features,
                                int32_t out_features, int32_t* flags, void* stream) {
    NFK_REQUIRE(Y || (y_hi_ && y_lo_), "no output requested");
    return linear_f16x3_launch(a_hi_, a_lo_, lda, a_exp, w_hi_, w_lo_, ldw, w_exp, bias, R, ldr, Y, ldy, y_hi_, y_lo_, lds, y_exp,
                               split_cols, y_first_col, relu_out, split_relu, n_rows, in_features, out_features, flags, stream, nullptr);
}

extern "C" int nfk_affine_coupling_final_f16x3(const void* a_hi, const void* a_lo, int64_t lda, int32_t a_exp, const void* w_hi,
                                               const void* w_lo, int64_t ldw, int32_t w_exp, const float* bias, int32_t hidden_features,
                                               const float* x, int64_t ldx, const int32_t* t_cols, int32_t t_col0, int32_t d_t,
                                               int32_t mult, int32_t scale_activation, int inverse, float* y, int64_t ldy,
                                               float* lad_accum, int64_t n_rows, int32_t* flags, void* stream) {
    NFK_REQUIRE(d_t >= 1 && (mult == 1 || mult == 2) && (scale_activation == 0 || scale_activation == 1), "bad coupling description");
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(x && y && (t_cols || t_col0 >= 0), "NULL pointer");
    CouplingEpilogue ce{x, ldx, y, ldy, t_cols, t_col0, d_t, mult, scale_activation, inverse, lad_accum};
    return linear_f16x3_launch(a_hi, a_lo, lda, a_exp, w_hi, w_lo, ldw, w_exp, bias, nullptr, 0, nullptr, 0, nullptr, nullptr, 0, 0, 0, 0,
                               0, 0, n_rows, hidden_features, mult * d_t, flags, stream, &ce);
}

static int linear_f16x3_launch(const void* a_hi_, const void* a_lo_, int64_t lda, int32_t a_exp, const void* w_hi_,
                               const void* w_lo_, int64_t ldw, int32_t w_exp, const float* bias, const float* R, int64_t ldr,
                               float* Y, int64_t ldy, void* y_hi_, void* y_lo_, int64_t lds, int32_t y_exp, int32_t split_cols,
                               int32_t y_first_col, int relu_out, int split_relu, int64_t n_rows, int32_t in_features,
                               int32_t out_features, int32_t* flags, void* stream, const CouplingEpilogue* ce) {
    const __half* a_hi = (const __half*)a_hi_; const __half* a_lo = (const __half*)a_lo_;
    const __half* w_hi = (const __half*)w_hi_; const __half* w_lo = (const __half*)w_lo_;
    __half* y_hi = (__half*)y_hi_; __half* y_lo = (__half*)y_lo_;
    NFK_REQUIRE(n_rows >= 0 && in_features >= 1 && out_features >= 1, "bad sizes");
    NFK_REQUIRE(act_valid(relu_out) && act_valid(split_relu), "unknown activation code (relu_out=%d, split_relu=%d)", relu_out, split_relu);
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(a_hi && a_lo && w_hi && w_lo, "NULL operand pointer");
    NFK_REQUIRE(ce || Y || (y_hi && y_lo), "no output requested");
    NFK_REQUIRE((y_hi == nullptr) == (y_lo == nullptr), "y_hi and y_lo must be given together");
    NFK_REQUIRE(nfk_linear_f16x3_supported(lda, ldw, in_features), "f16x3 path needs in_features, lda, ldw multiples of 8");
    NFK_REQUIRE(aligned16(a_hi) && aligned16(a_lo) && aligned16(w_hi) && aligned16(w_lo), "operands must be 16-byte aligned");
    NFK_REQUIRE(n_rows < (1ll << 31), "n_rows too large for one launch");
    NFK_REQUIRE(pow2_exp_ok(a_exp) && pow2_exp_ok(w_exp) && pow2_exp_ok(y_exp), "scale exponent out of range");

    tc::Params p;
    p.bias = bias; p.residual = R; p.y = Y; p.y_hi = y_hi; p.y_lo = y_lo; p.flags = flags;
    p.acc_scale = ldexpf(1.0f, a_exp + w_exp); p.inv_acc_scale = ldexpf(1.0f, -(a_exp + w_exp)); p.out_scale = ldexpf(1.0f, y_exp);
    p.split_n = split_cols > 0 ? split_cols : out_features;
    p.ldr = ldr; p.ldy = ldy; p.lds = lds; p.n_rows = n_rows; p.K = in_features; p.N = out_features;
    p.relu_out = relu_out; p.split_relu = split_relu;
    p.y_first_col = y_first_col > 0 ? y_first_col : 0;
    p.drain = tc::DRAIN_SLABS_LINEAR;
    p.cx = nullptr; p.cy = nullptr; p.c_cols = nullptr; p.c_lad = nullptr; p.ldcx = p.ldcy = 0;
    p.c_col0 = p.c_dt = p.c_mult = p.c_act = p.c_inverse = 0;
    if (ce) {
        p.cx = ce->x; p.cy = ce->y; p.c_cols = ce->t_cols; p.c_lad = ce->lad; p.ldcx = ce->ldx; p.ldcy = ce->ldy;
        p.c_col0 = ce->t_col0; p.c_dt = ce->d_t; p.c_mult = ce->mult; p.c_act = ce->act; p.c_inverse = ce->inverse;
    }
    p.num_n_tiles = (out_features + tc::BN - 1) / tc::BN;
    p.num_m_tiles = (int)((n_rows + tc::BM - 1) / tc::BM);
    CUtensorMap ma_hi, ma_lo, mw_hi, mw_lo;
    int rc;
    if ((rc = tc::make_map(&ma_hi, a_hi, n_rows, in_features, lda, tc::BM))) return rc;
    if ((rc = tc::make_map(&ma_lo, a_lo, n_rows, in_features, lda, tc::BM))) return rc;
    if ((rc = tc::make_map(&mw_hi, w_hi, out_features, in_features, ldw, tc::BN))) return rc;
    if ((rc = tc::make_map(&mw_lo, w_lo, out_features, in_features, ldw, tc::BN))) return rc;

    const bool act = relu_out > NFK_ACT_RELU || split_relu > NFK_ACT_RELU;
    static DeviceOnce attr_once[2];
    int attr_dev = 0;
    if (attr_once[act].pending(&attr_dev)) {
        cudaError_t e = cudaFuncSetAttribute(act ? tc::linear_f16x3_kernel<true> : tc::linear_f16x3_kernel<false>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, tc::LIN_SMEM_BYTES);
        if (e != cudaSuccess) return fail(NFK_E_CUDA, "cudaFuncSetAttribute(smem=%d): %s", tc::LIN_SMEM_BYTES, cudaGetErrorString(e));
        attr_once[act].mark(attr_dev);
    }
    const int64_t work = (int64_t)p.num_m_tiles * p.num_n_tiles;
    const int grid = (int)(work < tc::sm_count() ? work : tc::sm_count());
    if (act)
        tc::linear_f16x3_kernel<true><<<grid, tc::THREADS, tc::LIN_SMEM_BYTES, (cudaStream_t)stream>>>(ma_hi, ma_lo, mw_hi, mw_lo, p);
    else
        tc::linear_f16x3_kernel<false><<<grid, tc::THREADS, tc::LIN_SMEM_BYTES, (cudaStream_t)stream>>>(ma_hi, ma_lo, mw_hi, mw_lo, p);
    return check_launch("linear_f16x3_kernel");
}
