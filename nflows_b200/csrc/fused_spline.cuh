// Pieces shared by the tensor-core kernels that evaluate the rational-quadratic spline straight from their accumulators
// (nfk_rq_coupling_tc.cu: final conditioner layer + spline; nfk_coupling_step_tc.cu: the whole coupling step).
#pragma once
#include "rq_spline.cuh"
#include "tc_common.cuh"

namespace nfk {
namespace tc {

// The spline of rq_spline.cuh::rqs_eval for F features at once, IN PLACE on the accumulator registers
// v[f*MP + 0..M): [K widths | K heights | K-1 (tails) or K+1 derivatives].  Same formulas and operation order per
// feature; the f-loops are innermost so the F dependency chains interleave in the instruction stream.
template <int NB, bool TAILS, int F, int MP>
__device__ __forceinline__ void rqs_eval_multi(const SplineParams& p, bool inverse, const float (&xin)[F], float (&v)[F * MP],
                                               float (&y)[F], float (&lad)[F], int& flag) {
    bool inside[F];
    float x[F], mw[F], mh[F], sw[F], sh[F];
#pragma unroll
    for (int f = 0; f < F; ++f) {
        inside[f] = (xin[f] >= p.left) && (xin[f] <= p.right);
        if (!TAILS && !inside[f]) flag |= 1;
        x[f] = inside[f] ? xin[f] : (xin[f] > p.right ? p.right : p.left);
        mw[f] = v[f * MP];
        mh[f] = v[f * MP + NB];
    }
#pragma unroll
    for (int k = 1; k < NB; ++k)
#pragma unroll
        for (int f = 0; f < F; ++f) {
            mw[f] = fmaxf(mw[f], v[f * MP + k]);
            mh[f] = fmaxf(mh[f], v[f * MP + NB + k]);
        }
    const float c2 = p.pre_scale * 1.4426950408889634f;
#pragma unroll
    for (int f = 0; f < F; ++f) { sw[f] = 0.0f; sh[f] = 0.0f; }
#pragma unroll
    for (int k = 0; k < NB; ++k)
#pragma unroll
        for (int f = 0; f < F; ++f) {
            const float a = ex2_approx((v[f * MP + k] - mw[f]) * c2);
            const float b = ex2_approx((v[f * MP + NB + k] - mh[f]) * c2);
            v[f * MP + k] = a;
            v[f * MP + NB + k] = b;
            sw[f] += a;
            sh[f] += b;
        }
    float rw[F], rh[F], cum_w[F], cum_h[F], kw_lo[F], kh_lo[F], b_cw[F], b_ch[F], b_w[F], b_h[F];
    int bin[F];
#pragma unroll
    for (int f = 0; f < F; ++f) {
        rw[f] = fast_div(p.mix_w, sw[f]);
        rh[f] = fast_div(p.mix_h, sh[f]);
        cum_w[f] = 0.0f; cum_h[f] = 0.0f;
        kw_lo[f] = p.left; kh_lo[f] = p.bottom;
        b_cw[f] = p.left; b_ch[f] = p.bottom; b_w[f] = 1.0f; b_h[f] = 1.0f;
        bin[f] = 0;
    }
#pragma unroll
    for (int k = 0; k < NB; ++k)
#pragma unroll
        for (int f = 0; f < F; ++f) {
            cum_w[f] += fmaf(v[f * MP + k], rw[f], p.min_w);
            cum_h[f] += fmaf(v[f * MP + NB + k], rh[f], p.min_h);
            const float kw_hi = (k == NB - 1) ? p.right : fmaf(p.span_w, cum_w[f], p.left);
            const float kh_hi = (k == NB - 1) ? p.top : fmaf(p.span_h, cum_h[f], p.bottom);
            const bool take = (k == 0) || (x[f] >= (inverse ? kh_lo[f] : kw_lo[f]));
            bin[f] = take ? k : bin[f];
            b_cw[f] = take ? kw_lo[f] : b_cw[f];
            b_ch[f] = take ? kh_lo[f] : b_ch[f];
            b_w[f] = take ? kw_hi - kw_lo[f] : b_w[f];
            b_h[f] = take ? kh_hi - kh_lo[f] : b_h[f];
            kw_lo[f] = kw_hi; kh_lo[f] = kh_hi;
        }
    // derivative logits of the selected bin: d[k] for k = 0..NB with d[0] = d[NB] = edge (tails) else stored K+1 values
    float ud0[F], ud1[F];
#pragma unroll
    for (int f = 0; f < F; ++f) {
        ud0[f] = TAILS ? p.edge_ud : v[f * MP + 2 * NB];
        ud1[f] = TAILS ? (NB > 1 ? v[f * MP + 2 * NB] : p.edge_ud) : v[f * MP + 2 * NB + 1];
    }
#pragma unroll
    for (int k = 1; k < NB; ++k)
#pragma unroll
        for (int f = 0; f < F; ++f) {
            const float dk = TAILS ? v[f * MP + 2 * NB + k - 1] : v[f * MP + 2 * NB + k];
            const float dk1 = TAILS ? (k + 1 < NB ? v[f * MP + 2 * NB + k] : p.edge_ud) : v[f * MP + 2 * NB + k + 1];
            ud0[f] = (k == bin[f]) ? dk : ud0[f];
            ud1[f] = (k == bin[f]) ? dk1 : ud1[f];
        }
#pragma unroll
    for (int f = 0; f < F; ++f) {
        const float d0 = p.min_d + fast_softplus(ud0[f], p.beta, p.inv_beta);
        const float d1 = p.min_d + fast_softplus(ud1[f], p.beta, p.inv_beta);
        const float delta = fast_div(b_h[f], b_w[f]);
        const float s = d0 + d1 - 2.0f * delta;
        float theta, ys;
        if (inverse) {
            const float u = x[f] - b_ch[f];
            const float a = u * s + b_h[f] * (delta - d0);
            const float b = b_h[f] * d0 - u * s;
            const float c = -delta * u;
            const float disc = b * b - 4.0f * a * c;
            if (!(disc >= 0.0f)) flag |= 2;
            theta = fast_div(2.0f * c, -b - sqrtf(disc));
            ys = theta * b_w[f] + b_cw[f];
        } else {
            theta = fast_div(x[f] - b_cw[f], b_w[f]);
        }
        const float t1mt = theta * (1.0f - theta);
        const float den = delta + s * t1mt;
        if (!inverse) {
            const float num = b_h[f] * (delta * (theta * theta) + d0 * t1mt);
            ys = b_ch[f] + fast_div(num, den);
        }
        const float omt = 1.0f - theta;
        const float dnum = (delta * delta) * (d1 * (theta * theta) + 2.0f * delta * t1mt + d0 * (omt * omt));
        const float l = fast_log(dnum) - 2.0f * fast_log(den);
        const bool identity = TAILS && !inside[f];
        y[f] = identity ? xin[f] : ys;
        lad[f] = identity ? 0.0f : (inverse ? -l : l);
    }
}

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
