// Test infrastructure: host build of the per-element spline source of the row kernels (nflows_b200/csrc/rq_spline.cuh) --
// the forward nfk_rqs_rows evaluates and the vector-Jacobian product nfk_rqs_rows_backward evaluates -- exported through a small
// C ABI so tests/test_spline_training_host.py can check the backward's arithmetic against fp64 autograd without a GPU.
// Compiled by that test into a temporary directory (g++, contraction to FMA as nvcc does).
#include "../nflows_b200/csrc/rq_spline.cuh"

// Element e: x[e], parameters params[e*M .. e*M + M) in the row kernel's packed order.

// the forward of nfk_rqs_rows at the instance it dispatches to: the lean form for K = 8 / 16, the scan form otherwise
template <int KMAX, bool EXACT>
static void fwd_run(const nfk::SplineParams& p, bool inv, const float* x, const float* params, long long n, float* y, float* lad,
                    int& flag) {
    const int M = nfk::spline_param_count(p.num_bins, p.linear_tails);
    for (long long e = 0; e < n; ++e) {
        const float* q = params + e * M;
        auto at = [&](int i) { return q[i]; };
        if (EXACT) {
            nfk::rqs_eval_lean_one<KMAX>(p, inv, x[e], at, y[e], lad[e], flag);
        } else {
            float w[KMAX], h[KMAX], d[KMAX + 1];
            nfk::rqs_load_packed<KMAX, EXACT>(p, at, w, h, d);
            nfk::rqs_eval<KMAX, EXACT>(p, inv, x[e], w, h, d, y[e], lad[e], flag);
        }
    }
}

template <int KMAX, bool EXACT, bool LEAN>
static void vjp_run(const nfk::SplineParams& p, bool inv, const float* x, const float* params, const float* gy, const float* gl,
                    long long n, float* gx, float* gparams) {
    const int M = nfk::spline_param_count(p.num_bins, p.linear_tails);
    for (long long e = 0; e < n; ++e) {
        const float* q = params + e * M;
        float* g = gparams + e * M;
        float w[KMAX], h[KMAX], d[KMAX + 1];
        nfk::rqs_load_packed<KMAX, EXACT>(p, [&](int i) { return q[i]; }, w, h, d);
        nfk::rqs_vjp<KMAX, EXACT, LEAN>(p, inv, x[e], w, h, d, gy[e], gl[e], gx[e]);
        nfk::rqs_store_grads<KMAX, EXACT>(p, w, h, d, [&](int i, float v) { g[i] = v; });
    }
}

// per-element forward of the row kernel; -1 for a bin count without an instance
extern "C" int rqs_host_rows(const NfkSplineDesc* desc, int inverse, const float* x, const float* params, long long n, float* y,
                             float* lad, int* flags) {
    const nfk::SplineParams p = nfk::spline_params_of(*desc);
    const int K = p.num_bins;
    if (K < 1 || K > NFK_MAX_BINS) return -1;
    int flag = 0;
    nfk::with_bin_instance(K, [&](auto km, auto ex) { fwd_run<km, ex>(p, inverse != 0, x, params, n, y, lad, flag); });
    if (flags) *flags = flag;
    return 0;
}

// per-element VJP (cotangents gy[e], gl[e]) at the instance nfk_rqs_rows_backward dispatches to.  lean = 1: the knots with the
// lean form's arithmetic (what the kernel does for K = 8 / 16; -1 for other K); lean = 0: the scan form's arithmetic.
extern "C" int rqs_host_rows_vjp(const NfkSplineDesc* desc, int inverse, int lean, const float* x, const float* params,
                                 const float* gy, const float* gl, long long n, float* gx, float* gparams) {
    const nfk::SplineParams p = nfk::spline_params_of(*desc);
    const int K = p.num_bins;
    if (K < 1 || K > NFK_MAX_BINS) return -1;
    if (lean && K != 8 && K != 16) return -1;
    const bool inv = inverse != 0;
    nfk::with_bin_instance(K, [&](auto km, auto ex) {
        if (lean) vjp_run<km, ex, true>(p, inv, x, params, gy, gl, n, gx, gparams);
        else vjp_run<km, ex, false>(p, inv, x, params, gy, gl, n, gx, gparams);
    });
    return 0;
}
