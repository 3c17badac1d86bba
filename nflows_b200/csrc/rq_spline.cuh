// Rational-quadratic spline, one element per thread, everything in registers.
//
// Numerical contract (SURVEY.md Appendix A) = reference nflows/transforms/splines/rational_quadratic.py:13-181
// and nflows/utils/torchutils.py:134-136, restated for a thread that owns all K unnormalised widths/heights
// and the K+1 unnormalised derivatives of ONE element:
//   * softmax with max-subtraction and a true division, min-size mixing, sequential prefix sum, affine map to
//     [lo,hi], first/last knot forced (:91-98, :106-113);
//   * bin = last k in [0,K-1] with x >= knot_k (the reference counts x >= knot over all K+1 knots after adding
//     1e-6 to the last one; identical for in-domain x because knots are non-decreasing);
//   * only the two derivatives the bin needs go through softplus (threshold 20, like F.softplus);
//   * forward: theta=(x-cw)/w ...; inverse: root = 2c / (-b - sqrt(b^2-4ac)) (:132-181).
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#include <cuda_runtime.h>
#define NFK_HD __device__ __forceinline__
#else
#define NFK_HD static inline      // host build: oracle/rqs_host.cpp evaluates the SAME source on the CPU
#endif

#include "../../include/nfk.h"

namespace nfk {

struct SplineParams {        // derived on the host in double precision, rounded once to fp32 (like the
    int num_bins;            // Python-float -> fp32-scalar conversions the reference's tensor ops perform)
    int linear_tails;
    float left, right, bottom, top;
    float span_w, span_h;    // float(right-left), float(top-bottom)
    float min_w, min_h, min_d;
    float mix_w, mix_h;      // float(1 - min_w*K), float(1 - min_h*K)
    float beta, inv_beta;    // softplus beta
    float pre_scale;         // float(1/float(sqrt(H))): ATen divides by a CPU scalar as x * (1/s)
    float edge_ud;           // float(log(exp(1-min_d)-1)): boundary unnormalised derivative for linear tails
    float knot_eps;          // 1e-6f, searchsorted eps
};

// host: derive the fp32 constants from the descriptor (nfk_spline.cu)
int make_spline_params(const NfkSplineDesc* d, SplineParams* p);

NFK_HD float softplus_torch(float x, float beta, float inv_beta) {
    // F.softplus(x, beta, threshold=20): x*beta > 20 ? x : log1p(exp(x*beta))/beta
    float xb = x * beta;
    return xb > 20.0f ? x : log1pf(expf(xb)) * inv_beta;
}

NFK_HD float ex2_approx(float x) {
#ifdef __CUDA_ARCH__
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#else
    return exp2f(x);
#endif
}

// ---- cheap forms used on the epilogue critical path (NFK_SPLINE_FAST, default on).  Each replaces a ~10-30 instruction
// IEEE/libm sequence by 2-6 instructions with <= ~2 ulp (division, log) error; the per-element effect (~1e-7 relative)
// is below the fp32 round-off of the reference formulation (profiles/parity_calibration_*.txt, tests/test_kernel_source_on_host.py)
#ifndef NFK_SPLINE_FAST
#define NFK_SPLINE_FAST 1
#endif

NFK_HD float rcp_approx(float x) {                 // MUFU.RCP (<= 1 ulp), no range fix-ups
#ifdef __CUDA_ARCH__
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#else
    return 1.0f / x;
#endif
}

NFK_HD float lg2_approx(float x) {                 // MUFU.LG2
#ifdef __CUDA_ARCH__
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#else
    return log2f(x);
#endif
}

// a / b for operands far from the fp32 range limits (bin widths, interpolation denominators): one MUFU + one FMUL.
// (__fdividef wraps the same two instructions in ~10 more that rescale huge denominators; ncu r2: the spline epilogue is
// bound by instruction issue, 12 instructions per division.)
NFK_HD float fast_div(float a, float b) {
#if NFK_SPLINE_FAST
    return a * rcp_approx(b);
#else
    return a / b;
#endif
}

NFK_HD float fast_log(float x) {
#if NFK_SPLINE_FAST
    return lg2_approx(x) * 0.693147180559945f;     // __logf without its denormal rescaling: arguments here are >= ~1e-12
#else
    return logf(x);
#endif
}

// softplus with F.softplus semantics (beta, threshold 20) = max(z,0) + log1p(exp(-|z|)), z = beta*x
NFK_HD float fast_softplus(float x, float beta, float inv_beta) {
#if NFK_SPLINE_FAST
    const float z = x * beta;
    const float t = ex2_approx(-fabsf(z) * 1.4426950408889634f);             // exp(-|z|) in (0, 1]
    // log1p(t): short series where 1+t would lose the small t, MUFU log otherwise
    const float l = t < 0.0078125f ? t * (1.0f - t * (0.5f - t * 0.33333334f)) : fast_log(1.0f + t);
    const float sp = fmaxf(z, 0.0f) + l;
    return z > 20.0f ? x : sp * inv_beta;
#else
    return softplus_torch(x, beta, inv_beta);
#endif
}

// KMAX: compile-time bound on the number of bins (register arrays); p.num_bins <= KMAX.
// uw/uh: K raw values (before the 1/sqrt(H) pre-scale); ud: K+1 raw derivative logits (already padded with
// edge_ud for linear tails).  Returns y and log|dy/dx|; sets flag bits for domain / discriminant violations.
//
// Written branch-free (outside-the-tails elements are evaluated on a clamped input and discarded by a select) so
// that several elements of one thread can be interleaved by the scheduler, and with the cheap forms that keep the
// result inside the fp32 round-off of the reference: softmax as ex2((u - max) * log2e/sqrt(H)) (MUFU, rel. error
// <= 2^-22) normalised by ONE reciprocal per softmax instead of K divisions; the bin ratio, theta and the rational
// function keep IEEE divisions, logf/log1pf/expf of the two derivatives and of the log-determinant stay accurate.
// EXACT: the caller guarantees p.num_bins == KMAX, which lets every `k < K` guard fold away at compile time.
template <int KMAX, bool EXACT = false>
NFK_HD void rqs_eval(const SplineParams& p, bool inverse, float x_in, const float (&uw)[KMAX],
                                         const float (&uh)[KMAX], const float (&ud)[KMAX + 1], float& y, float& lad,
                                         int& flag) {
    const int K = EXACT ? KMAX : p.num_bins;
    const bool inside = (x_in >= p.left) && (x_in <= p.right);   // NaN -> outside (reference :26-39)
    if (!p.linear_tails && !inside) flag |= 1;                   // reference raises InputOutsideDomain (:81-82)
    const float x = inside ? x_in : (x_in > p.right ? p.right : p.left);

    float ew[KMAX], eh[KMAX];
    float mw = -INFINITY, mh = -INFINITY;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            mw = fmaxf(mw, uw[k]);
            mh = fmaxf(mh, uh[k]);
        }
    }
    const float c2 = p.pre_scale * 1.4426950408889634f;          // log2(e) / sqrt(H)
    float sw = 0.0f, sh = 0.0f;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            ew[k] = ex2_approx((uw[k] - mw) * c2);
            eh[k] = ex2_approx((uh[k] - mh) * c2);
            sw += ew[k];
            sh += eh[k];
        }
    }
    const float rw = fast_div(p.mix_w, sw), rh = fast_div(p.mix_h, sh);

    // running prefix sums -> knots; select the bin on the fly.  The instances for more than 16 bins compensate the sums
    // (Kahan): a plain float scan loses ~sqrt(K) ulp on the knots, and the knot error dominates the log|det| error at large K.
    // Measured on an H100 (700 W) with nfk_rqs_elementwise, 65536 elements of randn*2 logits (wh_divisor 4), error percentile
    // over that of the fp32 reference on CUDA's float cumsum, both against fp64: at K = 24..64, plain scan 1.2-1.5x at the
    // 99th / 99.9th percentile of y and log|det| (8192-element samples reached 2.6x at the 99.9th, K = 64 inverse), compensated
    // 0.9-1.2x; at K = 16 (plain scan) 1.1-1.4x.  Register use of the KMAX 32 / 64 instances is unchanged by the two carried
    // values (ptxas: 207 / 255 registers in the rows kernel, 216 / 255 in the elementwise kernel; the same spills).
    float cum_w = 0.0f, cum_h = 0.0f, err_w = 0.0f, err_h = 0.0f;
    float kw_lo = p.left, kh_lo = p.bottom;              // knot k
    float b_cw = p.left, b_ch = p.bottom, b_w = 1.0f, b_h = 1.0f;
    int bin = 0;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            if (KMAX > 16) {
                const float vw = fmaf(ew[k], rw, p.min_w) - err_w, tw = cum_w + vw;
                const float vh = fmaf(eh[k], rh, p.min_h) - err_h, th = cum_h + vh;
                err_w = (tw - cum_w) - vw;
                err_h = (th - cum_h) - vh;
                cum_w = tw;
                cum_h = th;
            } else {
                cum_w += fmaf(ew[k], rw, p.min_w);
                cum_h += fmaf(eh[k], rh, p.min_h);
            }
            const float kw_hi = (k == K - 1) ? p.right : fmaf(p.span_w, cum_w, p.left);   // knot k+1
            const float kh_hi = (k == K - 1) ? p.top : fmaf(p.span_h, cum_h, p.bottom);
            const bool take = (k == 0) || (x >= (inverse ? kh_lo : kw_lo));
            bin = take ? k : bin;
            b_cw = take ? kw_lo : b_cw;
            b_ch = take ? kh_lo : b_ch;
            b_w = take ? kw_hi - kw_lo : b_w;
            b_h = take ? kh_hi - kh_lo : b_h;
            kw_lo = kw_hi; kh_lo = kh_hi;
        }
    }

    float ud0 = ud[0], ud1 = ud[1];
#pragma unroll
    for (int k = 1; k < KMAX; ++k) {
        ud0 = (k == bin) ? ud[k] : ud0;
        ud1 = (k == bin) ? ud[k + 1] : ud1;
    }
    const float d0 = p.min_d + fast_softplus(ud0, p.beta, p.inv_beta);
    const float d1 = p.min_d + fast_softplus(ud1, p.beta, p.inv_beta);
    const float delta = fast_div(b_h, b_w);
    const float s = d0 + d1 - 2.0f * delta;

    float theta, ys;
    if (inverse) {
        const float u = x - b_ch;
        const float a = u * s + b_h * (delta - d0);
        const float b = b_h * d0 - u * s;
        const float c = -delta * u;
        const float disc = b * b - 4.0f * a * c;
        if (!(disc >= 0.0f)) flag |= 2;                   // reference: assert (discriminant >= 0).all() (:142)
        theta = fast_div(2.0f * c, -b - sqrtf(disc));
        ys = theta * b_w + b_cw;
    } else {
        theta = fast_div(x - b_cw, b_w);
    }
    const float t1mt = theta * (1.0f - theta);
    const float den = delta + s * t1mt;
    if (!inverse) {
        const float num = b_h * (delta * (theta * theta) + d0 * t1mt);
        ys = b_ch + fast_div(num, den);
    }
    const float omt = 1.0f - theta;
    const float dnum = (delta * delta) * (d1 * (theta * theta) + 2.0f * delta * t1mt + d0 * (omt * omt));
    const float l = fast_log(dnum) - 2.0f * fast_log(den);
    const bool identity = p.linear_tails && !inside;
    y = identity ? x_in : ys;
    lad = identity ? 0.0f : (inverse ? -l : l);
}

// ------------------------------------------------------------------------------------------------------------------------
// Lean evaluation of F features at once, IN PLACE on registers v[f*MP + 0..M): [NB widths | NB heights | NB-1 (tails) or NB+1
// derivative logits] -- the form the tensor-core epilogues and (F = 1) the HBM-bound row kernel use when the bin count is a
// compile-time constant.  Same formulas as rqs_eval; what is different is the instruction count (ncu r2: the spline was 624
// instructions per feature and the coupling-step kernel's epilogue warps, not its tensor pipe, set the pace):
//   * direction and tail mode are template parameters (no runtime selects between the forward and inverse formulas);
//   * softmax arguments are one FFMA each (v * c - max * c);
//   * all knots are formed first, then the bin is found by BINARY search over the register arrays -- log2(K) comparisons, each
//     followed by selects that halve the candidate knots / derivative logits -- instead of a K-step scan carrying five selects;
//   * divisions and logarithms are single MUFU operations (fast_div / fast_log above).
// The f-loops are innermost so the F dependency chains interleave in the instruction stream.
template <int NB, bool TAILS, bool INVERSE, int F, int MP>
NFK_HD void rqs_eval_lean(const SplineParams& p, const float (&xin)[F], float (&v)[F * MP], float (&y)[F], float (&lad)[F],
                          int& flag) {
    constexpr int P = NB <= 2 ? 2 : NB <= 4 ? 4 : NB <= 8 ? 8 : NB <= 16 ? 16 : NB <= 32 ? 32 : 64;   // search width
    bool inside[F];
    float x[F], mw[F], mh[F], sw[F], sh[F];
#pragma unroll
    for (int f = 0; f < F; ++f) {
        inside[f] = (xin[f] >= p.left) && (xin[f] <= p.right);   // NaN -> outside (reference :26-39)
        if (!TAILS && !inside[f]) flag |= 1;                     // reference raises InputOutsideDomain (:81-82)
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
    const float c2 = p.pre_scale * 1.4426950408889634f;          // log2(e) / sqrt(H)
#pragma unroll
    for (int f = 0; f < F; ++f) { mw[f] = -mw[f] * c2; mh[f] = -mh[f] * c2; sw[f] = 0.0f; sh[f] = 0.0f; }
#pragma unroll
    for (int k = 0; k < NB; ++k)
#pragma unroll
        for (int f = 0; f < F; ++f) {
            const float a = ex2_approx(fmaf(v[f * MP + k], c2, mw[f]));
            const float b = ex2_approx(fmaf(v[f * MP + NB + k], c2, mh[f]));
            v[f * MP + k] = a;
            v[f * MP + NB + k] = b;
            sw[f] += a;
            sh[f] += b;
        }
    // knots: prefix sums of the mixed bin sizes, mapped to [left, right] / [bottom, top], first and last forced (:91-98, :106-113)
    float kw[F][P + 1], kh[F][P + 1], dd[F][P + 1];
#pragma unroll
    for (int f = 0; f < F; ++f) {
        sw[f] = p.mix_w * rcp_approx(sw[f]);                     // from here on: the softmax normalisers
        sh[f] = p.mix_h * rcp_approx(sh[f]);
        mw[f] = 0.0f; mh[f] = 0.0f;                              // ... and the running sums
        kw[f][0] = p.left; kh[f][0] = p.bottom;
    }
#pragma unroll
    for (int k = 0; k < NB; ++k)
#pragma unroll
        for (int f = 0; f < F; ++f) {
            mw[f] += fmaf(v[f * MP + k], sw[f], p.min_w);
            mh[f] += fmaf(v[f * MP + NB + k], sh[f], p.min_h);
            kw[f][k + 1] = (k == NB - 1) ? p.right : fmaf(p.span_w, mw[f], p.left);
            kh[f][k + 1] = (k == NB - 1) ? p.top : fmaf(p.span_h, mh[f], p.bottom);
        }
#pragma unroll
    for (int k = 0; k <= P; ++k)
#pragma unroll
        for (int f = 0; f < F; ++f) {
            if (k > NB) { kw[f][k] = INFINITY; kh[f][k] = INFINITY; }           // padding of the search: never taken
            // padded search (K not a power of two): the last real knot is compared at an inner level, where x == last knot
            // must still fall into the last bin -- the searched array carries +inf there and gets the constant back below
            if (P != NB && k == NB) { if (INVERSE) kh[f][k] = INFINITY; else kw[f][k] = INFINITY; }
            // derivative logit at knot k: the boundary constant for linear tails, else the stored K+1 values
            dd[f][k] = k > NB ? 0.0f : (TAILS ? ((k == 0 || k == NB) ? p.edge_ud : v[f * MP + 2 * NB + k - 1]) : v[f * MP + 2 * NB + k]);
        }
    // binary search for the last knot <= x (x is inside [first, last] knot by now): halve the candidates log2(P) times
#pragma unroll
    for (int width = P; width > 1; width >>= 1) {
        const int h = width >> 1;
#pragma unroll
        for (int f = 0; f < F; ++f) {
            const bool up = x[f] >= (INVERSE ? kh[f][h] : kw[f][h]);
#pragma unroll
            for (int i = 0; i <= h; ++i) {
                kw[f][i] = up ? kw[f][h + i] : kw[f][i];
                kh[f][i] = up ? kh[f][h + i] : kh[f][i];
                dd[f][i] = up ? dd[f][h + i] : dd[f][i];
            }
        }
    }
#pragma unroll
    for (int f = 0; f < F; ++f) {
        if (P != NB) {
            if (INVERSE) kh[f][1] = kh[f][1] == INFINITY ? p.top : kh[f][1];
            else kw[f][1] = kw[f][1] == INFINITY ? p.right : kw[f][1];
        }
        const float b_cw = kw[f][0], b_w = kw[f][1] - kw[f][0];
        const float b_ch = kh[f][0], b_h = kh[f][1] - kh[f][0];
        const float d0 = p.min_d + fast_softplus(dd[f][0], p.beta, p.inv_beta);
        const float d1 = p.min_d + fast_softplus(dd[f][1], p.beta, p.inv_beta);
        const float delta = fast_div(b_h, b_w);
        const float s = d0 + d1 - 2.0f * delta;
        float theta, ys;
        if (INVERSE) {
            const float u = x[f] - b_ch;
            const float a = u * s + b_h * (delta - d0);
            const float b = b_h * d0 - u * s;
            const float c = -delta * u;
            const float disc = b * b - 4.0f * a * c;
            if (!(disc >= 0.0f)) flag |= 2;                   // reference: assert (discriminant >= 0).all() (:142)
            theta = fast_div(2.0f * c, -b - sqrtf(disc));
            ys = theta * b_w + b_cw;
        } else {
            theta = fast_div(x[f] - b_cw, b_w);
        }
        const float t1mt = theta * (1.0f - theta);
        const float den = delta + s * t1mt;
        if (!INVERSE) {
            const float num = b_h * (delta * (theta * theta) + d0 * t1mt);
            ys = b_ch + fast_div(num, den);
        }
        const float omt = 1.0f - theta;
        const float dnum = (delta * delta) * (d1 * (theta * theta) + 2.0f * delta * t1mt + d0 * (omt * omt));
        const float l = fast_log(dnum) - 2.0f * fast_log(den);
        const bool identity = TAILS && !inside[f];
        y[f] = identity ? xin[f] : ys;
        lad[f] = identity ? 0.0f : (INVERSE ? -l : l);
    }
}

}  // namespace nfk
