// Pieces shared by the tensor-core kernels that evaluate the rational-quadratic spline straight from their accumulators
// (nfk_rq_coupling_tc.cu: final conditioner layer + spline; nfk_coupling_step_tc.cu: the whole coupling step).
#pragma once
#include "rq_spline.cuh"
#include "tc_common.cuh"

namespace nfk {
namespace tc {

// Column tile of the final conditioner layer: the packed weight has MP = roundup(M, 8) rows per transformed feature (zero
// padded), a tile of TF * MP <= BN packed rows holds whole features, and after the MMAs every consumer thread PAIR owns one
// row: each thread evaluates FPT = TF / 2 features of it.
template <int NB, bool TAILS>
struct FusedCfg {
    static constexpr int M = TAILS ? 3 * NB - 1 : 3 * NB + 1;   // parameters per feature
    static constexpr int MP = (M + 7) / 8 * 8;                  // padded
    static constexpr int FPT = BN / (2 * MP);                   // features per thread (two threads per row)
    static constexpr int TF = 2 * FPT;                          // features per column tile
    static constexpr int TILE = TF * MP;                        // packed weight rows per column tile (<= BN)
    static_assert(FPT >= 1, "unsupported bin count for the fused kernels");
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

// A consumer warpgroup's 64 x 128 sums (wgmma fragment layout, tc_common.cuh: wgmma_f16) -> stg[64][ld], row-major.
__device__ __forceinline__ void stage_sums(float* stg, int ld, const float (&sum)[64], int wi, int lane) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
            *reinterpret_cast<float2*>(stg + (wi * 16 + (lane >> 2) + 8 * h) * ld + 8 * j + 2 * (lane & 3)) =
                make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
}

// Thread (row, half fh) of column tile n: its FPT features back from the power-of-two scaled domain plus the packed bias,
// the spline, the output (fp32 y or its fp16 pair) and the row's log|det| share (lad_row).  srow: the row's staged sums.
template <int NB, bool TAILS>
__device__ __forceinline__ void spline_tile(const SplineOut& o, const float* srow, int n, int64_t row, bool row_ok, int fh,
                                            float& lad_row, int& flag) {
    using Cfg = FusedCfg<NB, TAILS>;
    constexpr int MP = Cfg::MP, FPT = Cfg::FPT, TF = Cfg::TF, TILE = Cfg::TILE;
    const int j0 = n * TF + fh * FPT;                   // first feature this thread owns in this tile
    float v[FPT * MP];
    const float* s = srow + fh * FPT * MP;
    const float* b = o.bias + (int64_t)n * TILE + fh * FPT * MP;
#pragma unroll
    for (int c = 0; c < FPT * MP; ++c) v[c] = fmaf(s[c], o.inv_acc_scale, (j0 + c / MP < o.d_t) ? __ldg(b + c) : 0.0f);
    float xin[FPT];
    int col[FPT];
#pragma unroll
    for (int f = 0; f < FPT; ++f) {
        const bool ok = row_ok && (j0 + f < o.d_t);
        col[f] = !ok ? 0 : (o.t_cols ? __ldg(o.t_cols + j0 + f) : o.t_col0 + j0 + f);
        xin[f] = ok ? o.x[row * o.ldx + col[f]] : 0.0f;
    }
    // all FPT features advanced together (ILP = FPT)
    float yy[FPT], ll[FPT];
    if (o.inverse) rqs_eval_lean<NB, TAILS, true, FPT, MP>(o.sp, xin, v, yy, ll, flag);
    else rqs_eval_lean<NB, TAILS, false, FPT, MP>(o.sp, xin, v, yy, ll, flag);
#pragma unroll
    for (int f = 0; f < FPT; ++f) {
        if (!(row_ok && j0 + f < o.d_t)) continue;
        lad_row += ll[f];
        if (o.y_hi) {
            __half hi, lo;
            split_f16(yy[f], o.out_scale, hi, lo, flag);
            o.y_hi[row * o.lds + col[f]] = hi;
            o.y_lo[row * o.lds + col[f]] = lo;
        } else {
            o.y[row * o.ldy + col[f]] = yy[f];
        }
    }
}

}  // namespace tc
}  // namespace nfk
