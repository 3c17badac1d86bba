// Pieces shared by the tensor-core kernels that evaluate the rational-quadratic spline straight from their accumulators
// (nfk_rq_coupling_tc.cu: final conditioner layer + spline; nfk_coupling_step_tc.cu: the whole coupling step).
#pragma once
#include "rq_spline.cuh"
#include "tc_common.cuh"

namespace nfk {
namespace tc {

// NB = AFFINE_NB selects the affine epilogue of the masked autoregressive transform instead of the spline (reference
// transforms/autoregressive.py:96-128): M = MP = 2 parameters per feature, MADE's rows 2j, 2j + 1 = (u_j, shift_j) with no
// padding, scale_j = softplus(u_j) + 1e-3.  A 128-row column tile then holds 64 whole features, 32 per thread.
constexpr int AFFINE_NB = 0;

// NB = mog_nb(MP) < 0 selects the mixture-of-Gaussians epilogue of MixtureOfGaussiansMADE (reference nn/nde/made.py:284-427):
// MADE's 3C rows (logit, mean, unconstrained std) of each feature packed to MP = -8 NB rows, zero padded.  The component count
// C <= MP / 3 is a runtime argument (MogOut), so one instance serves every C that packs to the same MP.
constexpr int mog_nb(int mp) { return -mp / 8; }

// Column tile of the final conditioner layer: the packed weight has MP = roundup(M, 8) rows per transformed feature (zero
// padded), a tile of TF * MP <= BN packed rows holds whole features, and after the MMAs every consumer thread PAIR owns one
// row: each thread evaluates FPT = TF / 2 features of it.
template <int NB, bool TAILS>
struct FusedCfg {
    static constexpr bool AFFINE = NB == AFFINE_NB;
    static constexpr bool MOG = NB < 0;
    static constexpr int M = AFFINE ? 2 : (MOG ? -8 * NB : (TAILS ? 3 * NB - 1 : 3 * NB + 1));   // parameters per feature
    static constexpr int MP = AFFINE ? 2 : (M + 7) / 8 * 8;                  // padded
    static constexpr int FPT = BN / (2 * MP);                   // features per thread (two threads per row)
    static constexpr int TF = 2 * FPT;                          // features per column tile
    static constexpr int TILE = TF * MP;                        // packed weight rows per column tile (<= BN)
    static constexpr int LD = (TILE + 31) / 32 * 32;            // staged row stride in floats of a TILE-wide MMA (stg_chunk:
                                                                // whole groups of 8 chunks; 96 at TILE = 96, else 128)
    static_assert(FPT >= 1, "unsupported bin count for the fused kernels");
    static_assert(!(AFFINE && TAILS), "the affine epilogue has no tails");
    static_assert(!MOG || (!TAILS && MP <= 64), "mixture epilogue: no tails, at most 64 rows per feature");
};

// What the mixture epilogue reads besides SplineOut (nfk_mog_made_step_f16x3, include/nfk.h: NfkMogArgs).
struct MogOut {
    const float* u;         // sample: uniforms [n_rows, ldn] (feature j in column j), else null
    const float* e;         // sample: standard normals, same layout
    int64_t ldn;
    float eps;              // std = softplus(unconstrained) + eps
    int C;                  // mixture components, 3C <= MP
    int sample;             // 0: log_prob into lad_accum, 1: draw y
};

// What the spline epilogue reads and writes.
struct SplineOut {
    const float* bias;      // [d_t * MP] packed like the weight rows, zero padded
    const float* x;         // coupling input [n_rows, ldx]
    float* y;               // coupling output [n_rows, ldy] (transformed columns only), or null when the pair is written
    __half* y_hi;           // fp16 split pair of the outputs [n_rows, lds] (the consumer is a tensor-core layer), or null
    __half* y_lo;
    const int32_t* t_cols;  // [d_t] column of transformed feature j, or null: feature j lives in column t_col0 + j
    int t_col0;
    float out_scale;        // 2^e of the pair output
    int64_t ldx, ldy, lds;
    int d_t;
    int inverse;
    float inv_acc_scale;    // 2^-(e_a + e_w): the accumulators hold (A Wp^T) * 2^(e_a + e_w)
    SplineParams sp;
};

// Staged sums of one 64-row pass: stg[64][LD] floats (LD = BN, or FusedCfg::LD for TILE-wide MMAs), row-major, each row's
// 16-byte chunks permuted so that both sides of the staging are free of bank conflicts.  The permutation stays within aligned
// groups of 8 chunks, and a row stride of a multiple of 32 floats keeps every row on the same bank alignment.  Logical chunk c (columns 4c .. 4c + 3) of row r sits at chunk c ^ g(r) ^ s(c):
//   * g(r) in {0, 3, 5, 6} for r % 4 = 0 .. 3.  The fragment stores (8 bytes, a half-warp = 4 rows x 2 chunks of the same
//     column pair) then differ in bits 1-2 between rows and in bit 0 within a row: 16 distinct 8-byte bank pairs.  The row reads
//     (16 bytes, 8 threads = 4 rows x 2 feature halves) differ in bits 0-1 between rows;
//   * s(c) = 4 for the second feature half when its first chunk C = FPT * MP / 4 is a multiple of 8, so that the two halves of a
//     row, read at the same step, differ in bit 2 (C = 12 already does; C = 14, bins = 16 without tails, keeps a 2-way conflict).
template <int NB, bool TAILS>
__device__ __forceinline__ int stg_chunk(int r, int c) {
    constexpr int C = FusedCfg<NB, TAILS>::FPT * FusedCfg<NB, TAILS>::MP / 4;
    return c ^ ((0x6530 >> (4 * (r & 3))) & 7) ^ ((C % 8 == 0 && c >= C) ? 4 : 0);
}

// A consumer warpgroup's 64 x N sums (wgmma fragment layout, tc_common.cuh: wgmma_f16) -> stg (layout above, row stride LD).
template <int NB, bool TAILS, int N, int LD = BN>
__device__ __forceinline__ void stage_sums(float* stg, const float (&sum)[N / 2], int wi, int lane) {
    static_assert(N <= LD && LD % 32 == 0, "staged row stride");
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wi * 16 + (lane >> 2) + 8 * h, c = 2 * j + ((lane & 3) >> 1);
            *reinterpret_cast<float2*>(stg + r * LD + 4 * stg_chunk<NB, TAILS>(r, c) + 2 * (lane & 1)) =
                make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
        }
}

// The coupling inputs of thread (row, half fh) in column tile n and the output columns they go to.  Loaded before the tile's
// MMAs are waited for, so that their latency hides behind them.  The affine epilogue's features are consecutive columns
// (t_cols is NULL): it keeps no column list, and its 32 inputs are loaded by the epilogue itself (affine_tile).
template <int NB, bool TAILS>
struct SplineIn {
    float x[FusedCfg<NB, TAILS>::FPT];
    int col[FusedCfg<NB, TAILS>::FPT];
};
template <bool TAILS>
struct SplineIn<AFFINE_NB, TAILS> {};
template <int NB, bool TAILS>
__device__ __forceinline__ SplineIn<NB, TAILS> spline_inputs(const SplineOut& o, int n, int64_t row, bool row_ok, int fh) {
    constexpr int FPT = FusedCfg<NB, TAILS>::FPT, TF = FusedCfg<NB, TAILS>::TF;
    SplineIn<NB, TAILS> in;
    if constexpr (!FusedCfg<NB, TAILS>::AFFINE) {
        const int j0 = n * TF + fh * FPT;
#pragma unroll
        for (int f = 0; f < FPT; ++f) {
            const bool ok = row_ok && (j0 + f < o.d_t) && (!FusedCfg<NB, TAILS>::MOG || o.x != nullptr);   // mixture draws: no x
            in.col[f] = !ok ? 0 : (o.t_cols ? __ldg(o.t_cols + j0 + f) : o.t_col0 + j0 + f);
            in.x[f] = ok ? o.x[row * o.ldx + in.col[f]] : 0.0f;
        }
    }
    return in;
}

// The packed bias of column tile n (TILE floats) into the shared-memory buffer dst by cp.async, zero past d_t * MP: threads
// t < TILE / 4 of a warpgroup copy 16 bytes each (MP is a multiple of 8, so no chunk straddles d_t * MP).  The copies land
// once the issuing threads have passed cp_async_wait_all; a barrier after that makes them visible to the other threads.
// The affine epilogue's features are 2 floats each: threads t < TILE / 2 copy 8 bytes (one feature) each.
template <int NB, bool TAILS>
__device__ __forceinline__ void bias_tile_async(float* dst, const SplineOut& o, int n, int t) {
    constexpr int TILE = FusedCfg<NB, TAILS>::TILE, MP = FusedCfg<NB, TAILS>::MP;
    if constexpr (FusedCfg<NB, TAILS>::AFFINE) {
        if (t < TILE / 2) {
            const int e = n * TILE + 2 * t;
            const uint32_t bytes = e < o.d_t * MP ? 8u : 0u;
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(dst + 2 * t)), "l"(o.bias + (bytes ? e : 0)),
                         "r"(bytes)
                         : "memory");
        }
    } else if (t < TILE / 4) {
        const int e = n * TILE + 4 * t;
        const uint32_t bytes = e < o.d_t * MP ? 16u : 0u;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst + 4 * t)), "l"(o.bias + (bytes ? e : 0)),
                     "r"(bytes)
                     : "memory");
    }
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Thread (row, half fh) of column tile n: its FPT features back from the power-of-two scaled domain plus the packed bias,
// the spline, the output (fp32 y or its fp16 pair) and the row's log|det| share (lad_row).  stg: the staged sums (row stride
// LD), r: the row within them.  BIAS_SMEM: the tile's packed bias is read from bias_tile in shared memory (bias_tile_async),
// else from o.bias.
// The affine epilogue of thread (row, half fh) of column tile n (reference transforms/autoregressive.py:96-128): its FPT features
// j = t_col0 + j0 + f from (u_j, shift_j), scale_j = softplus(u_j) + 1e-3 as F.softplus computes it (threshold 20, accurate
// expf / log1pf), y_j = scale_j * x_j + shift_j (inverse: (x_j - shift_j) / scale_j, IEEE division), each operation rounded on
// its own like the reference's tensor ops; lad_row += (inverse ? -1 : 1) * sum_j log(scale_j), in feature order.  fp32 output.
template <int NB, bool TAILS, int LD, bool BIAS_SMEM>
__device__ __forceinline__ void affine_tile(const SplineOut& o, const float* stg, int r, int n, int64_t row, bool row_ok, int fh,
                                            float& lad_row, const float* bias_tile) {
    using Cfg = FusedCfg<NB, TAILS>;
    constexpr int FPT = Cfg::FPT, TF = Cfg::TF, TILE = Cfg::TILE, C = FPT * 2 / 4;
    const int j0 = n * TF + fh * FPT;
    const int64_t c0 = (int64_t)o.t_col0 + j0;
    const float* b = o.bias + (int64_t)n * TILE + fh * FPT * 2;
    float lad = 0.0f;
    // G features at a time: their inputs are loaded together (the stores to y stop later loads from moving ahead of them)
    constexpr int G = 8;
#pragma unroll
    for (int g = 0; g < FPT; g += G) {
        float x[G];
#pragma unroll
        for (int f = 0; f < G; ++f) x[f] = (row_ok && j0 + g + f < o.d_t) ? __ldg(o.x + row * o.ldx + c0 + g + f) : 0.0f;
#pragma unroll
        for (int i = g / 2; i < (g + G) / 2; ++i) {     // chunk i: features 2 i, 2 i + 1 of this thread
            const float4 s = *reinterpret_cast<const float4*>(stg + r * LD + 4 * stg_chunk<NB, TAILS>(r, fh * C + i));
            const float sv[4] = {s.x, s.y, s.z, s.w};
            float bv[4];
            if constexpr (BIAS_SMEM) {                  // zero past d_t * 2 already
                const float4 bq = *reinterpret_cast<const float4*>(bias_tile + fh * FPT * 2 + 4 * i);
                bv[0] = bq.x; bv[1] = bq.y; bv[2] = bq.z; bv[3] = bq.w;
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) bv[e] = (j0 + 2 * i + e / 2 < o.d_t) ? __ldg(b + 4 * i + e) : 0.0f;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int f = 2 * i + h;
                if (!(row_ok && j0 + f < o.d_t)) continue;
                const float u = fmaf(sv[2 * h], o.inv_acc_scale, bv[2 * h]);
                const float shift = fmaf(sv[2 * h + 1], o.inv_acc_scale, bv[2 * h + 1]);
                const float scale = __fadd_rn(softplus_torch(u, 1.0f, 1.0f), 1e-3f);
                const float xf = x[f - g];
                const float y = o.inverse ? __fdiv_rn(__fsub_rn(xf, shift), scale) : __fadd_rn(__fmul_rn(scale, xf), shift);
                o.y[row * o.ldy + c0 + f] = y;
                lad = __fadd_rn(lad, logf(scale));
            }
        }
    }
    lad_row += o.inverse ? -lad : lad;
}

// The mixture epilogue of thread (row, half fh) of column tile n (reference nn/nde/made.py:333-401).  Feature j's rows
// (3c, 3c + 1, 3c + 2) = (logit l_c, mean mu_c, unconstrained std u_c), sigma_c = softplus(u_c) + eps (threshold 20, accurate
// expf / log1pf), log-softmax and logsumexp max-subtracted as torch computes them:
//   log_prob: lad_row += sum_j LSE_c( log_softmax(l)_c - 0.5 (log 2 pi + 2 log sigma_c + ((x_j - mu_c) / sigma_c)^2) ),
//             the features in order;
//   sample:   c* = the first c with u_j < sum_{c' <= c} softmax(l)_{c'} (C - 1 when rounding leaves u_j above the total),
//             y_j = mu_{c*} + sigma_{c*} e_j (fp32).
// The bias comes from the tile's copy in shared memory (bias_tile_async).
template <int NB, bool TAILS, int LD>
__device__ __forceinline__ void mog_tile(const SplineOut& o, const MogOut& g, const float* stg, int r, int n, int64_t row, bool row_ok,
                                         int fh, const SplineIn<NB, TAILS>& in, float& lad_row, const float* bias_tile) {
    using Cfg = FusedCfg<NB, TAILS>;
    constexpr int MP = Cfg::MP, FPT = Cfg::FPT, TF = Cfg::TF, C4 = FPT * MP / 4, CMAX = MP / 3;
    constexpr float LOG_2PI = 1.8378770664093453f;
    const int j0 = n * TF + fh * FPT;
    float v[FPT * MP];
#pragma unroll
    for (int i = 0; i < C4; ++i) {
        const float4 s = *reinterpret_cast<const float4*>(stg + r * LD + 4 * stg_chunk<NB, TAILS>(r, fh * C4 + i));
        const float4 bq = *reinterpret_cast<const float4*>(bias_tile + fh * FPT * MP + 4 * i);
        v[4 * i + 0] = fmaf(s.x, o.inv_acc_scale, bq.x);
        v[4 * i + 1] = fmaf(s.y, o.inv_acc_scale, bq.y);
        v[4 * i + 2] = fmaf(s.z, o.inv_acc_scale, bq.z);
        v[4 * i + 3] = fmaf(s.w, o.inv_acc_scale, bq.w);
    }
    float lp = 0.0f;
#pragma unroll
    for (int f = 0; f < FPT; ++f) {
        if (!(row_ok && j0 + f < o.d_t)) continue;
        const float* q = v + f * MP;
        float lmax = -INFINITY;
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < g.C) lmax = fmaxf(lmax, q[3 * c]);
        float se = 0.0f;
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < g.C) se = __fadd_rn(se, expf(__fsub_rn(q[3 * c], lmax)));
        const int64_t col = (int64_t)o.t_col0 + j0 + f;
        if (!g.sample) {
            const float lse = logf(se), x = in.x[f];
            float t[CMAX];
            float tmax = -INFINITY;
#pragma unroll
            for (int c = 0; c < CMAX; ++c) {
                if (c >= g.C) continue;
                const float sigma = __fadd_rn(softplus_torch(q[3 * c + 2], 1.0f, 1.0f), g.eps);
                const float z = __fdiv_rn(__fsub_rn(x, q[3 * c + 1]), sigma);
                const float quad = __fadd_rn(__fadd_rn(LOG_2PI, __fmul_rn(2.0f, logf(sigma))), __fmul_rn(z, z));
                t[c] = __fsub_rn(__fsub_rn(__fsub_rn(q[3 * c], lmax), lse), __fmul_rn(0.5f, quad));
                tmax = fmaxf(tmax, t[c]);
            }
            float st = 0.0f;
#pragma unroll
            for (int c = 0; c < CMAX; ++c)
                if (c < g.C) st = __fadd_rn(st, expf(__fsub_rn(t[c], tmax)));
            lp = __fadd_rn(lp, __fadd_rn(logf(st), tmax));
        } else {
            const float uu = __ldg(g.u + row * g.ldn + j0 + f), ee = __ldg(g.e + row * g.ldn + j0 + f);
            float cum = 0.0f, mu = 0.0f, us = 0.0f;
            bool found = false;
#pragma unroll
            for (int c = 0; c < CMAX; ++c) {
                if (c >= g.C) continue;
                cum = __fadd_rn(cum, __fdiv_rn(expf(__fsub_rn(q[3 * c], lmax)), se));
                if (!found && (uu < cum || c == g.C - 1)) {
                    found = true;
                    mu = q[3 * c + 1];
                    us = q[3 * c + 2];
                }
            }
            const float sigma = __fadd_rn(softplus_torch(us, 1.0f, 1.0f), g.eps);
            o.y[row * o.ldy + col] = __fadd_rn(mu, __fmul_rn(ee, sigma));
        }
    }
    lad_row += lp;
}

template <int NB, bool TAILS, int LD = BN, bool BIAS_SMEM = false>
__device__ __forceinline__ void spline_tile(const SplineOut& o, const float* stg, int r, int n, int64_t row, bool row_ok, int fh,
                                            const SplineIn<NB, TAILS>& in, float& lad_row, int& flag,
                                            const float* bias_tile = nullptr) {
    using Cfg = FusedCfg<NB, TAILS>;
    if constexpr (Cfg::AFFINE) {
        affine_tile<NB, TAILS, LD, BIAS_SMEM>(o, stg, r, n, row, row_ok, fh, lad_row, bias_tile);
    } else {
        constexpr int MP = Cfg::MP, FPT = Cfg::FPT, TF = Cfg::TF, TILE = Cfg::TILE, C = FPT * MP / 4;
        const int j0 = n * TF + fh * FPT;                   // first feature this thread owns in this tile
        float v[FPT * MP];
        const float* b = o.bias + (int64_t)n * TILE + fh * FPT * MP;
#pragma unroll
        for (int i = 0; i < C; ++i) {
            const float4 s = *reinterpret_cast<const float4*>(stg + r * LD + 4 * stg_chunk<NB, TAILS>(r, fh * C + i));
            const float sv[4] = {s.x, s.y, s.z, s.w};
            if constexpr (BIAS_SMEM) {                      // zero past d_t * MP already
                const float4 bq = *reinterpret_cast<const float4*>(bias_tile + fh * FPT * MP + 4 * i);
                const float bv[4] = {bq.x, bq.y, bq.z, bq.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) v[4 * i + e] = fmaf(sv[e], o.inv_acc_scale, bv[e]);
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int c = 4 * i + e;
                    v[c] = fmaf(sv[e], o.inv_acc_scale, (j0 + c / MP < o.d_t) ? __ldg(b + c) : 0.0f);
                }
            }
        }
        // all FPT features advanced together (ILP = FPT)
        float yy[FPT], ll[FPT];
        if (o.inverse) rqs_eval_lean<NB, TAILS, true, FPT, MP>(o.sp, in.x, v, yy, ll, flag);
        else rqs_eval_lean<NB, TAILS, false, FPT, MP>(o.sp, in.x, v, yy, ll, flag);
#pragma unroll
        for (int f = 0; f < FPT; ++f) {
            if (!(row_ok && j0 + f < o.d_t)) continue;
            lad_row += ll[f];
            if (o.y_hi) {
                __half hi, lo;
                split_f16(yy[f], o.out_scale, hi, lo, flag);
                o.y_hi[row * o.lds + in.col[f]] = hi;
                o.y_lo[row * o.lds + in.col[f]] = lo;
            } else {
                o.y[row * o.ldy + in.col[f]] = yy[f];
            }
        }
    }
}

}  // namespace tc
}  // namespace nfk
