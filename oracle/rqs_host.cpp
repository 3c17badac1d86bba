// TEST INFRASTRUCTURE.  Host build of nflows_b200/csrc/rq_spline.cuh: the exact source the CUDA kernels evaluate per
// element, compiled for the CPU (ex2.approx -> exp2f), exported through a tiny C ABI so tests can study the numerics of
// the kernel formulation against the fp64 oracle without a GPU.  Built by oracle/Makefile into oracle/_build/.
#include <string.h>

#include "../nflows_b200/csrc/rq_spline.cuh"

namespace nfk {
int make_spline_params_host(const NfkSplineDesc* d, SplineParams* p) {
    const int K = d->num_bins;
    p->num_bins = K;
    p->linear_tails = d->linear_tails ? 1 : 0;
    p->left = (float)d->left; p->right = (float)d->right; p->bottom = (float)d->bottom; p->top = (float)d->top;
    p->span_w = (float)(d->right - d->left);
    p->span_h = (float)(d->top - d->bottom);
    p->min_w = (float)d->min_bin_width; p->min_h = (float)d->min_bin_height; p->min_d = (float)d->min_derivative;
    p->mix_w = (float)(1.0 - d->min_bin_width * K);
    p->mix_h = (float)(1.0 - d->min_bin_height * K);
    p->beta = (float)d->softplus_beta;
    p->inv_beta = (float)(1.0 / d->softplus_beta);
    float div = (float)d->wh_divisor;
    p->pre_scale = (d->wh_divisor == 1.0) ? 1.0f : (float)(1.0 / (double)div);
    p->edge_ud = (float)log(exp(1.0 - d->min_derivative) - 1.0);
    p->knot_eps = 1e-6f;
    return 0;
}
}  // namespace nfk

// rqs_eval at one instance, loading the parameters as rqs_elementwise_kernel does (zeros past K, edge_ud for linear tails)
template <int KMAX, bool EXACT>
static void scan_run(const nfk::SplineParams& p, bool inverse, const float* x, const float* uw, const float* uh, const float* ud,
                     long long n, float* y, float* lad, int& flag) {
    const int K = p.num_bins;
    const int nd = p.linear_tails ? K - 1 : K + 1;
    for (long long e = 0; e < n; ++e) {
        float w[KMAX], h[KMAX], d[KMAX + 1];
        for (int k = 0; k < KMAX; ++k) {
            w[k] = k < K ? uw[e * K + k] : 0.0f;
            h[k] = k < K ? uh[e * K + k] : 0.0f;
        }
        if (p.linear_tails) {
            for (int k = 0; k <= KMAX; ++k) d[k] = (k >= 1 && k < K) ? ud[e * nd + k - 1] : p.edge_ud;
        } else {
            for (int k = 0; k <= KMAX; ++k) d[k] = k <= K ? ud[e * nd + k] : 0.0f;
        }
        nfk::rqs_eval<KMAX, EXACT>(p, inverse, x[e], w, h, d, y[e], lad[e], flag);
    }
}

// The instances nfk_rqs_elementwise dispatches to (nfk_spline.cu), chosen by the same rule; -1 for K outside [1, NFK_MAX_BINS].
extern "C" int rqs_host_eval(const NfkSplineDesc* desc, int inverse, const float* x, const float* uw, const float* uh,
                             const float* ud, long long n, float* y, float* lad, int* flags) {
    nfk::SplineParams p;
    nfk::make_spline_params_host(desc, &p);
    const int K = p.num_bins;
    if (K < 1 || K > NFK_MAX_BINS) return -1;
    int flag = 0;
    const bool inv = inverse != 0;
    if (K == 8) scan_run<8, true>(p, inv, x, uw, uh, ud, n, y, lad, flag);
    else if (K < 8) scan_run<8, false>(p, inv, x, uw, uh, ud, n, y, lad, flag);
    else if (K == 16) scan_run<16, true>(p, inv, x, uw, uh, ud, n, y, lad, flag);
    else if (K < 16) scan_run<16, false>(p, inv, x, uw, uh, ud, n, y, lad, flag);
    else if (K <= 32) scan_run<32, false>(p, inv, x, uw, uh, ud, n, y, lad, flag);
    else scan_run<64, false>(p, inv, x, uw, uh, ud, n, y, lad, flag);
    if (flags) *flags = flag;
    return 0;
}

// The lean multi-feature form (rqs_eval_lean): F = 2 features per call, parameters packed as the kernels hold them.
template <int NB, bool TAILS, bool INV>
static void lean_run(const nfk::SplineParams& p, const float* x, const float* uw, const float* uh, const float* ud, long long n,
                     float* y, float* lad, int& flag) {
    constexpr int M = TAILS ? 3 * NB - 1 : 3 * NB + 1;
    constexpr int MP = (M + 7) / 8 * 8;
    constexpr int ND = TAILS ? NB - 1 : NB + 1;
    for (long long e = 0; e < n; e += 2) {
        float v[2 * MP] = {0};
        float xin[2] = {0, 0}, yy[2], ll[2];
        for (int f = 0; f < 2 && e + f < n; ++f) {
            xin[f] = x[e + f];
            for (int k = 0; k < NB; ++k) { v[f * MP + k] = uw[(e + f) * NB + k]; v[f * MP + NB + k] = uh[(e + f) * NB + k]; }
            for (int k = 0; k < ND; ++k) v[f * MP + 2 * NB + k] = ud[(e + f) * ND + k];
        }
        int fl = 0;
        nfk::rqs_eval_lean<NB, TAILS, INV, 2, MP>(p, xin, v, yy, ll, fl);
        for (int f = 0; f < 2 && e + f < n; ++f) { y[e + f] = yy[f]; lad[e + f] = ll[f]; }
        if (e + 1 < n || true) flag |= fl;      // (the pad element of an odd tail is x = 0 with zero logits: inside, no flag)
    }
}

extern "C" int rqs_host_eval_lean(const NfkSplineDesc* desc, int inverse, const float* x, const float* uw, const float* uh,
                                  const float* ud, long long n, float* y, float* lad, int* flags) {
    nfk::SplineParams p;
    nfk::make_spline_params_host(desc, &p);
    int flag = 0;
#define LEAN(NB)                                                                                    \
    if (p.num_bins == NB) {                                                                         \
        if (p.linear_tails) { if (inverse) lean_run<NB, true, true>(p, x, uw, uh, ud, n, y, lad, flag); else lean_run<NB, true, false>(p, x, uw, uh, ud, n, y, lad, flag); } \
        else { if (inverse) lean_run<NB, false, true>(p, x, uw, uh, ud, n, y, lad, flag); else lean_run<NB, false, false>(p, x, uw, uh, ud, n, y, lad, flag); } \
        if (flags) *flags = flag;                                                                   \
        return 0;                                                                                   \
    }
    LEAN(4) LEAN(8) LEAN(10) LEAN(16)
#undef LEAN
    return -1;
}
