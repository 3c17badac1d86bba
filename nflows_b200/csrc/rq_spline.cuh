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

#include <type_traits>

#ifdef __CUDACC__
#include <cuda_runtime.h>
#define NFK_HD __device__ __forceinline__
#define NFK_HOST_HD __host__ __device__ __forceinline__
#else
#define NFK_HD static inline      // host build: oracle/rqs_host.cpp evaluates the SAME source on the CPU
#define NFK_HOST_HD static inline
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

// host: validate the descriptor and derive the fp32 constants from it (nfk_spline.cu)
int make_spline_params(const NfkSplineDesc* d, SplineParams* p);

// The fp32 constants of a descriptor, without validation: make_spline_params checks the descriptor first, the host builds of
// this source call it directly.
inline SplineParams spline_params_of(const NfkSplineDesc& d) {
    SplineParams p;
    const int K = d.num_bins;
    p.num_bins = K;
    p.linear_tails = d.linear_tails ? 1 : 0;
    p.left = (float)d.left; p.right = (float)d.right; p.bottom = (float)d.bottom; p.top = (float)d.top;
    p.span_w = (float)(d.right - d.left);
    p.span_h = (float)(d.top - d.bottom);
    p.min_w = (float)d.min_bin_width; p.min_h = (float)d.min_bin_height; p.min_d = (float)d.min_derivative;
    p.mix_w = (float)(1.0 - d.min_bin_width * K);
    p.mix_h = (float)(1.0 - d.min_bin_height * K);
    p.beta = (float)d.softplus_beta;
    p.inv_beta = (float)(1.0 / d.softplus_beta);
    // x /= np.sqrt(H) on a tensor is executed by ATen as x * float(1.0 / float(sqrt(H)))
    const float div = (float)d.wh_divisor;
    p.pre_scale = (d.wh_divisor == 1.0) ? 1.0f : (float)(1.0 / (double)div);
    p.edge_ud = (float)log(exp(1.0 - d.min_derivative) - 1.0);
    p.knot_eps = 1e-6f;
    return p;
}

// M, the raw parameters of one element: [K widths | K heights | K - 1 (linear tails) or K + 1 derivative logits]
NFK_HOST_HD constexpr int spline_param_count(int K, int linear_tails) { return linear_tails ? 3 * K - 1 : 3 * K + 1; }

// The template instance that evaluates K bins, as (KMAX, EXACT): (8, exact) at K = 8, (8, scan) below 8, (16, exact) at 16,
// (16, scan) below 16, (32, scan) up to 32, else (64, scan).  Calls fn(std::integral_constant<int, KMAX>,
// std::integral_constant<bool, EXACT>) and returns what it returns.
template <class Fn>
inline auto with_bin_instance(int K, Fn&& fn) {
    using std::integral_constant;
    if (K == 8) return fn(integral_constant<int, 8>(), std::true_type());
    if (K < 8) return fn(integral_constant<int, 8>(), std::false_type());
    if (K == 16) return fn(integral_constant<int, 16>(), std::true_type());
    if (K < 16) return fn(integral_constant<int, 16>(), std::false_type());
    if (K <= 32) return fn(integral_constant<int, 32>(), std::false_type());
    return fn(integral_constant<int, 64>(), std::false_type());
}

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

// theta of the inverse: the root 2c / (-b - sqrt(b^2 - 4ac)) of the bin's quadratic (reference :132-146).  For an input inside
// the bin the discriminant is >= 0 and theta in [0, 1] in exact arithmetic.  At the top of a bin the discriminant is h^2 d1^2:
// with a flat bin (d1 near min_derivative) that is the difference of two terms ~4 h^2 delta^2 up to 1e6 times larger, and
// rounding alone takes it below zero (inputs on the height knots of a bin with derivative logits of -30, K = 10) or theta past 1.
// So a discriminant below zero by at most 1e-6 of the terms' magnitude (~8 ulp) counts as 0, and theta is clamped to [0, 1]
// (the clamp changes nothing where theta already lies there, nor a NaN).  A discriminant further below zero, or NaN, sets flag bit 2, as
// the reference's assertion (discriminant >= 0).all() (:142) would fail.
NFK_HD float inverse_theta(float a, float b, float c, int& flag) {
    const float disc = b * b - 4.0f * a * c;
    if (!(disc >= -1e-6f * (b * b + fabsf(4.0f * a * c)))) flag |= 2;
    const float theta = fast_div(2.0f * c, -b - sqrtf(fmaxf(disc, 0.0f)));
    return theta > 1.0f ? 1.0f : (theta < 0.0f ? 0.0f : theta);     // NaN and -0 pass unchanged
}

// The registers rqs_eval and rqs_vjp take, filled from one element's raw parameters: width k at uw(k), height k at uh(k) and
// derivative logit k at ud(k), k from 0; entries past K are 0, and linear tails put edge_ud at both ends of d.  Each accessor keeps
// its call site's index arithmetic (its width decides the kernels' code).
template <int KMAX, bool EXACT, class W, class H, class D>
NFK_HD void rqs_load(const SplineParams& p, W uw, H uh, D ud, float (&w)[KMAX], float (&h)[KMAX], float (&d)[KMAX + 1]) {
    const int K = EXACT ? KMAX : p.num_bins;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        w[k] = (k < K) ? uw(k) : 0.0f;
        h[k] = (k < K) ? uh(k) : 0.0f;
    }
    if (p.linear_tails) {
#pragma unroll
        for (int k = 0; k <= KMAX; ++k) d[k] = (k >= 1 && k < K) ? ud(k - 1) : p.edge_ud;
    } else {
#pragma unroll
        for (int k = 0; k <= KMAX; ++k) d[k] = (k <= K) ? ud(k) : 0.0f;
    }
}

// rqs_load from one packed run of M parameters, entry i at at(i)
template <int KMAX, bool EXACT, class At>
NFK_HD void rqs_load_packed(const SplineParams& p, At at, float (&w)[KMAX], float (&h)[KMAX], float (&d)[KMAX + 1]) {
    const int K = EXACT ? KMAX : p.num_bins;
    rqs_load<KMAX, EXACT>(p, [&](int k) { return at(k); }, [&](int k) { return at(K + k); }, [&](int k) { return at(2 * K + k); },
                          w, h, d);
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
        theta = inverse_theta(a, b, c, flag);
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
            theta = inverse_theta(a, b, c, flag);
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

// rqs_eval_lean of one element whose M packed parameters are read through at(i), direction and tail mode chosen at run time:
// the form the EXACT (p.num_bins == NB) instances of the HBM-bound kernels evaluate.
template <int NB, class At>
NFK_HD void rqs_eval_lean_one(const SplineParams& p, int inverse, float x, At at, float& y, float& lad, int& flag) {
    constexpr int MPL = spline_param_count(NB, false);
    float v[MPL];
    const float xin[1] = {x};
    float y1[1], l1[1];
    if (p.linear_tails) {
#pragma unroll
        for (int k = 0; k < spline_param_count(NB, true); ++k) v[k] = at(k);
        if (inverse) rqs_eval_lean<NB, true, true, 1, MPL>(p, xin, v, y1, l1, flag);
        else rqs_eval_lean<NB, true, false, 1, MPL>(p, xin, v, y1, l1, flag);
    } else {
#pragma unroll
        for (int k = 0; k < MPL; ++k) v[k] = at(k);
        if (inverse) rqs_eval_lean<NB, false, true, 1, MPL>(p, xin, v, y1, l1, flag);
        else rqs_eval_lean<NB, false, false, 1, MPL>(p, xin, v, y1, l1, flag);
    }
    y = y1[0];
    lad = l1[0];
}

// ------------------------------------------------------------------------------------------------------------------------
// Vector-Jacobian product of one element (training): given the element's input x_in, its raw parameters (uw, uh: K values
// before the 1/sqrt(H) pre-scale; ud: K+1 derivative logits, padded with edge_ud for linear tails, as rqs_eval takes them) and
// the cotangents gy of the output and gl of the log-determinant, returns g_x and overwrites uw, uh, ud IN PLACE with the
// gradients of the raw parameters (ud[0] and ud[K] of linear tails are the padding constants: the caller drops them).
// Nothing of the forward is saved: the knots are rebuilt from the parameters and the chain rule is applied by hand.
//   * bin: found exactly as by the forward instance this pairs with -- LEAN = the exponent arithmetic of rqs_eval_lean (the
//     EXACT K = 8 / 16 instances of the row kernel), else that of rqs_eval (with the compensated sums above 16 bins);
//   * forward map in bin k, theta = (x - cw)/w, delta = h/w, s = d0 + d1 - 2 delta, t = theta (1 - theta):
//       y = ch + h (delta theta^2 + d0 t) / den,  den = delta + s t
//       l = log(delta^2 D) - 2 log den,           D = d1 theta^2 + 2 delta t + d0 (1 - theta)^2
//     partials with respect to (theta, delta, d0, d1, h, ch), then theta_x = 1/w, theta_cw = -1/w, theta_w = -theta/w,
//     delta_h = 1/w, delta_w = -delta/w;
//   * knots: cw = knot k, w = knot k+1 - knot k; knot j = lo + span * sum_{i<j} size_i for 0 < j < K, the first and last knot
//     are forced (no gradient, as the reference's in-place assignment gives); size_i = min + mix softmax(pre_scale u)_i;
//   * derivatives: d = min_d + softplus(u; beta), softplus' = sigmoid(beta u), 1 above the threshold 20 (F.softplus);
//   * inverse (x = f^-1(z), L = -l(x)): the forward partials at the recovered theta with cotangents (-c, -gl),
//     c = (gy - gl l_x) / f_x, and g_z = c -- the implicit gradient of the root formula;
//   * linear tails outside [left, right]: identity, g_x = gy and every parameter gradient 0.
template <int KMAX, bool EXACT, bool LEAN>
NFK_HD void rqs_vjp(const SplineParams& p, bool inverse, float x_in, float (&uw)[KMAX], float (&uh)[KMAX], float (&ud)[KMAX + 1],
                    float gy, float gl, float& gx) {
    const int K = EXACT ? KMAX : p.num_bins;
    const bool inside = (x_in >= p.left) && (x_in <= p.right);
    const float x = inside ? x_in : (x_in > p.right ? p.right : p.left);

    float mw = -INFINITY, mh = -INFINITY;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            mw = fmaxf(mw, uw[k]);
            mh = fmaxf(mh, uh[k]);
        }
    }
    const float c2 = p.pre_scale * 1.4426950408889634f;
    const float nmw = -mw * c2, nmh = -mh * c2;
    float sw = 0.0f, sh = 0.0f;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {                       // uw, uh now hold the unnormalised softmax terms
        if (k < K) {
            uw[k] = ex2_approx(LEAN ? fmaf(uw[k], c2, nmw) : (uw[k] - mw) * c2);
            uh[k] = ex2_approx(LEAN ? fmaf(uh[k], c2, nmh) : (uh[k] - mh) * c2);
            sw += uw[k];
            sh += uh[k];
        }
    }
    const float rw = LEAN ? p.mix_w * rcp_approx(sw) : fast_div(p.mix_w, sw);
    const float rh = LEAN ? p.mix_h * rcp_approx(sh) : fast_div(p.mix_h, sh);

    float cum_w = 0.0f, cum_h = 0.0f, err_w = 0.0f, err_h = 0.0f;
    float kw_lo = p.left, kh_lo = p.bottom;
    float b_cw = p.left, b_ch = p.bottom, b_w = 1.0f, b_h = 1.0f;
    int bin = 0;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            if (KMAX > 16) {
                const float vw = fmaf(uw[k], rw, p.min_w) - err_w, tw = cum_w + vw;
                const float vh = fmaf(uh[k], rh, p.min_h) - err_h, th = cum_h + vh;
                err_w = (tw - cum_w) - vw;
                err_h = (th - cum_h) - vh;
                cum_w = tw;
                cum_h = th;
            } else {
                cum_w += fmaf(uw[k], rw, p.min_w);
                cum_h += fmaf(uh[k], rh, p.min_h);
            }
            const float kw_hi = (k == K - 1) ? p.right : fmaf(p.span_w, cum_w, p.left);
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

    float theta;
    if (inverse) {
        const float u = x - b_ch;
        const float a = u * s + b_h * (delta - d0);
        const float b = b_h * d0 - u * s;
        const float c = -delta * u;
        int no_flag = 0;                                   // the forward already raised what the inverse's root raises
        theta = inverse_theta(a, b, c, no_flag);
    } else {
        theta = fast_div(x - b_cw, b_w);
    }
    const float t = theta * (1.0f - theta);
    const float omt = 1.0f - theta;
    const float den = delta + s * t;
    const float num = delta * (theta * theta) + d0 * t;             // y = ch + h num / den
    const float dd = d1 * (theta * theta) + 2.0f * delta * t + d0 * (omt * omt);
    const float r_den = 1.0f / den, r_dd = 1.0f / dd, r_w = 1.0f / b_w;
    const float hr2 = b_h * r_den * r_den;
    const float one_m2th = 1.0f - 2.0f * theta, one_m2t = 1.0f - 2.0f * t;
    // local partials of y and l
    const float y_th = hr2 * delta * dd;                           // = w dy/dx
    const float l_th = 2.0f * (d1 * theta + delta * one_m2th - d0 * omt) * r_dd - 2.0f * s * one_m2th * r_den;
    const float y_de = hr2 * ((theta * theta) * den - num * one_m2t);
    const float l_de = 2.0f / delta + 2.0f * t * r_dd - 2.0f * one_m2t * r_den;
    const float y_d0 = hr2 * t * (den - num), y_d1 = -hr2 * num * t;
    const float l_d0 = (omt * omt) * r_dd - 2.0f * t * r_den, l_d1 = (theta * theta) * r_dd - 2.0f * t * r_den;

    // cotangents of the forward map at theta (inverse: (-c, -gl), c the gradient of the inverse's input)
    float GY = gy, GL = gl, g_in;
    if (inverse) {
        const float c = (gy * b_w - gl * l_th) / y_th;
        GY = -c;
        GL = -gl;
        g_in = c;
    }
    const float G_th = GY * y_th + GL * l_th;
    const float G_de = GY * y_de + GL * l_de;
    if (!inverse) g_in = G_th * r_w;
    const float g_cw = -G_th * r_w;
    const float g_w = -(G_th * theta + G_de * delta) * r_w;
    const float g_h = GY * num * r_den + G_de * r_w;
    const float g_ch = GY;
    const float z0 = ud0 * p.beta, z1 = ud1 * p.beta;
    const float g_d0 = (GY * y_d0 + GL * l_d0) * (z0 > 20.0f ? 1.0f : 1.0f / (1.0f + expf(-z0)));
    const float g_d1 = (GY * y_d1 + GL * l_d1) * (z1 > 20.0f ? 1.0f : 1.0f / (1.0f + expf(-z1)));

    // knots k and k + 1 -> bin sizes -> softmax logits: size_i collects the gradient of every free knot j > i
    const float gkw_lo = bin == 0 ? 0.0f : p.span_w * (g_cw - g_w), gkw_hi = bin == K - 1 ? 0.0f : p.span_w * g_w;
    const float gkh_lo = bin == 0 ? 0.0f : p.span_h * (g_ch - g_h), gkh_hi = bin == K - 1 ? 0.0f : p.span_h * g_h;
    float pw_lt = 0.0f, ph_lt = 0.0f;                              // softmax mass of the bins below `bin`
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K && k < bin) { pw_lt += uw[k]; ph_lt += uh[k]; }
    }
    float pw_bin = uw[0], ph_bin = uh[0];
#pragma unroll
    for (int k = 1; k < KMAX; ++k) {
        pw_bin = (k == bin) ? uw[k] : pw_bin;
        ph_bin = (k == bin) ? uh[k] : ph_bin;
    }
    const float inv_sw = 1.0f / sw, inv_sh = 1.0f / sh;
    const float tw = (gkw_lo * pw_lt + gkw_hi * (pw_lt + pw_bin)) * inv_sw;   // sum_i p_i G_i
    const float th = (gkh_lo * ph_lt + gkh_hi * (ph_lt + ph_bin)) * inv_sh;
    const float qw = p.pre_scale * p.mix_w * inv_sw, qh = p.pre_scale * p.mix_h * inv_sh;
    const bool identity = p.linear_tails && !inside;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            const float Gw = (k < bin ? gkw_lo : 0.0f) + (k <= bin ? gkw_hi : 0.0f);
            const float Gh = (k < bin ? gkh_lo : 0.0f) + (k <= bin ? gkh_hi : 0.0f);
            uw[k] = identity ? 0.0f : qw * uw[k] * (Gw - tw);
            uh[k] = identity ? 0.0f : qh * uh[k] * (Gh - th);
        }
    }
#pragma unroll
    for (int k = 0; k <= KMAX; ++k) ud[k] = identity ? 0.0f : (k == bin ? g_d0 : (k == bin + 1 ? g_d1 : 0.0f));
    gx = identity ? gy : g_in;
}

// Hands the parameter gradients rqs_vjp left in (w, h, d) to put(i, g), i the entry's index in the packed run of M; linear tails
// drop d[0] and d[K], the gradients of the padding constants.
template <int KMAX, bool EXACT, class Put>
NFK_HD void rqs_store_grads(const SplineParams& p, const float (&w)[KMAX], const float (&h)[KMAX], const float (&d)[KMAX + 1],
                            Put put) {
    const int K = EXACT ? KMAX : p.num_bins;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
            put(k, w[k]);
            put(K + k, h[k]);
        }
    }
    if (p.linear_tails) {
#pragma unroll
        for (int k = 1; k < KMAX; ++k)
            if (k < K) put(2 * K + k - 1, d[k]);
    } else {
#pragma unroll
        for (int k = 0; k <= KMAX; ++k)
            if (k <= K) put(2 * K + k, d[k]);
    }
}

}  // namespace nfk
