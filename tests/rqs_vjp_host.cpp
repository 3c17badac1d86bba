// Test infrastructure: host build of the per-element spline source of the row kernels (nflows_b200/csrc/rq_spline.cuh) --
// the forward nfk_rqs_rows evaluates and the vector-Jacobian product nfk_rqs_rows_backward evaluates -- exported through a small
// C ABI so tests/test_spline_training_host.py can check the backward's arithmetic against fp64 autograd without a GPU.
// Compiled by that test into a temporary directory (g++, contraction to FMA as nvcc does).
#include "../nflows_b200/csrc/rq_spline.cuh"

static nfk::SplineParams host_params(const NfkSplineDesc* d) {
    nfk::SplineParams p;
    const int K = d->num_bins;
    p.num_bins = K;
    p.linear_tails = d->linear_tails ? 1 : 0;
    p.left = (float)d->left; p.right = (float)d->right; p.bottom = (float)d->bottom; p.top = (float)d->top;
    p.span_w = (float)(d->right - d->left);
    p.span_h = (float)(d->top - d->bottom);
    p.min_w = (float)d->min_bin_width; p.min_h = (float)d->min_bin_height; p.min_d = (float)d->min_derivative;
    p.mix_w = (float)(1.0 - d->min_bin_width * K);
    p.mix_h = (float)(1.0 - d->min_bin_height * K);
    p.beta = (float)d->softplus_beta;
    p.inv_beta = (float)(1.0 / d->softplus_beta);
    const float div = (float)d->wh_divisor;
    p.pre_scale = (d->wh_divisor == 1.0) ? 1.0f : (float)(1.0 / (double)div);
    p.edge_ud = (float)log(exp(1.0 - d->min_derivative) - 1.0);
    p.knot_eps = 1e-6f;
    return p;
}

// element e: x[e], parameters params[e*M .. e*M + M) in the row kernel's order [K widths | K heights | K-1 or K+1 derivatives]
template <int KMAX>
static void load(const nfk::SplineParams& p, const float* q, float (&w)[KMAX], float (&h)[KMAX], float (&d)[KMAX + 1]) {
    const int K = p.num_bins;
    for (int k = 0; k < KMAX; ++k) {
        w[k] = k < K ? q[k] : 0.0f;
        h[k] = k < K ? q[K + k] : 0.0f;
    }
    for (int k = 0; k <= KMAX; ++k) {
        if (p.linear_tails) d[k] = (k >= 1 && k < K) ? q[2 * K + k - 1] : p.edge_ud;
        else d[k] = k <= K ? q[2 * K + k] : 0.0f;
    }
}

// the forward of nfk_rqs_rows at the instance it dispatches to: the lean form for K = 8 / 16, the scan form otherwise
template <int KMAX, bool EXACT>
static void fwd_run(const nfk::SplineParams& p, bool inv, const float* x, const float* params, long long n, float* y, float* lad,
                    int& flag) {
    const int K = p.num_bins, M = p.linear_tails ? 3 * K - 1 : 3 * K + 1;
    for (long long e = 0; e < n; ++e) {
        const float* q = params + e * M;
        if (EXACT) {
            constexpr int MPL = 3 * KMAX + 1;
            float v[MPL] = {0};
            for (int k = 0; k < M; ++k) v[k] = q[k];
            const float xin[1] = {x[e]};
            float y1[1], l1[1];
            if (p.linear_tails) {
                if (inv) nfk::rqs_eval_lean<KMAX, true, true, 1, MPL>(p, xin, v, y1, l1, flag);
                else nfk::rqs_eval_lean<KMAX, true, false, 1, MPL>(p, xin, v, y1, l1, flag);
            } else {
                if (inv) nfk::rqs_eval_lean<KMAX, false, true, 1, MPL>(p, xin, v, y1, l1, flag);
                else nfk::rqs_eval_lean<KMAX, false, false, 1, MPL>(p, xin, v, y1, l1, flag);
            }
            y[e] = y1[0];
            lad[e] = l1[0];
        } else {
            float w[KMAX], h[KMAX], d[KMAX + 1];
            load<KMAX>(p, q, w, h, d);
            nfk::rqs_eval<KMAX, false>(p, inv, x[e], w, h, d, y[e], lad[e], flag);
        }
    }
}

template <int KMAX, bool EXACT, bool LEAN>
static void vjp_run(const nfk::SplineParams& p, bool inv, const float* x, const float* params, const float* gy, const float* gl,
                    long long n, float* gx, float* gparams) {
    const int K = p.num_bins, M = p.linear_tails ? 3 * K - 1 : 3 * K + 1;
    for (long long e = 0; e < n; ++e) {
        float w[KMAX], h[KMAX], d[KMAX + 1];
        load<KMAX>(p, params + e * M, w, h, d);
        nfk::rqs_vjp<KMAX, EXACT, LEAN>(p, inv, x[e], w, h, d, gy[e], gl[e], gx[e]);
        float* g = gparams + e * M;
        for (int k = 0; k < K; ++k) { g[k] = w[k]; g[K + k] = h[k]; }
        if (p.linear_tails) for (int k = 1; k < K; ++k) g[2 * K + k - 1] = d[k];
        else for (int k = 0; k <= K; ++k) g[2 * K + k] = d[k];
    }
}

// per-element forward of the row kernel; -1 for a bin count without an instance
extern "C" int rqs_host_rows(const NfkSplineDesc* desc, int inverse, const float* x, const float* params, long long n, float* y,
                             float* lad, int* flags) {
    const nfk::SplineParams p = host_params(desc);
    const int K = p.num_bins;
    if (K < 1 || K > NFK_MAX_BINS) return -1;
    int flag = 0;
    const bool inv = inverse != 0;
    if (K == 8) fwd_run<8, true>(p, inv, x, params, n, y, lad, flag);
    else if (K < 8) fwd_run<8, false>(p, inv, x, params, n, y, lad, flag);
    else if (K == 16) fwd_run<16, true>(p, inv, x, params, n, y, lad, flag);
    else if (K < 16) fwd_run<16, false>(p, inv, x, params, n, y, lad, flag);
    else if (K <= 32) fwd_run<32, false>(p, inv, x, params, n, y, lad, flag);
    else fwd_run<64, false>(p, inv, x, params, n, y, lad, flag);
    if (flags) *flags = flag;
    return 0;
}

// per-element VJP (cotangents gy[e], gl[e]) at the instance nfk_rqs_rows_backward dispatches to.  lean = 1: the knots with the
// lean form's arithmetic (what the kernel does for K = 8 / 16; -1 for other K); lean = 0: the scan form's arithmetic.
extern "C" int rqs_host_rows_vjp(const NfkSplineDesc* desc, int inverse, int lean, const float* x, const float* params,
                                 const float* gy, const float* gl, long long n, float* gx, float* gparams) {
    const nfk::SplineParams p = host_params(desc);
    const int K = p.num_bins;
    if (K < 1 || K > NFK_MAX_BINS) return -1;
    if (lean && K != 8 && K != 16) return -1;
    const bool inv = inverse != 0;
    if (K == 8) {
        if (lean) vjp_run<8, true, true>(p, inv, x, params, gy, gl, n, gx, gparams);
        else vjp_run<8, true, false>(p, inv, x, params, gy, gl, n, gx, gparams);
    } else if (K < 8) vjp_run<8, false, false>(p, inv, x, params, gy, gl, n, gx, gparams);
    else if (K == 16) {
        if (lean) vjp_run<16, true, true>(p, inv, x, params, gy, gl, n, gx, gparams);
        else vjp_run<16, true, false>(p, inv, x, params, gy, gl, n, gx, gparams);
    } else if (K < 16) vjp_run<16, false, false>(p, inv, x, params, gy, gl, n, gx, gparams);
    else if (K <= 32) vjp_run<32, false, false>(p, inv, x, params, gy, gl, n, gx, gparams);
    else vjp_run<64, false, false>(p, inv, x, params, gy, gl, n, gx, gparams);
    return 0;
}
