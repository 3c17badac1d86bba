// TEST INFRASTRUCTURE.  Host build of nflows_b200/csrc/rq_spline.cuh: the exact source the CUDA kernels evaluate per
// element, compiled for the CPU (ex2.approx -> exp2f), exported through a tiny C ABI so tests can study the numerics of
// the kernel formulation against the fp64 oracle without a GPU.  Built by oracle/Makefile into oracle/_build/.
#include <string.h>

#include "../nflows_b200/csrc/rq_spline.cuh"

// rqs_eval at one instance, loading the parameters as rqs_elementwise_kernel does
template <int KMAX, bool EXACT>
static void scan_run(const nfk::SplineParams& p, bool inverse, const float* x, const float* uw, const float* uh, const float* ud,
                     long long n, float* y, float* lad, int& flag) {
    const int K = p.num_bins;
    const int nd = nfk::spline_param_count(K, p.linear_tails) - 2 * K;
    for (long long e = 0; e < n; ++e) {
        float w[KMAX], h[KMAX], d[KMAX + 1];
        nfk::rqs_load<KMAX, EXACT>(p, [&](int k) { return uw[e * K + k]; }, [&](int k) { return uh[e * K + k]; },
                                   [&](int k) { return ud[e * nd + k]; }, w, h, d);
        nfk::rqs_eval<KMAX, EXACT>(p, inverse, x[e], w, h, d, y[e], lad[e], flag);
    }
}

// The instances nfk_rqs_elementwise dispatches to (nfk_spline.cu), chosen by the same rule; -1 for K outside [1, NFK_MAX_BINS].
extern "C" int rqs_host_eval(const NfkSplineDesc* desc, int inverse, const float* x, const float* uw, const float* uh,
                             const float* ud, long long n, float* y, float* lad, int* flags) {
    const nfk::SplineParams p = nfk::spline_params_of(*desc);
    const int K = p.num_bins;
    if (K < 1 || K > NFK_MAX_BINS) return -1;
    int flag = 0;
    nfk::with_bin_instance(K, [&](auto km, auto ex) { scan_run<km, ex>(p, inverse != 0, x, uw, uh, ud, n, y, lad, flag); });
    if (flags) *flags = flag;
    return 0;
}

// The lean multi-feature form (rqs_eval_lean): F = 2 features per call, parameters packed as the kernels hold them.
template <int NB, bool TAILS, bool INV>
static void lean_run(const nfk::SplineParams& p, const float* x, const float* uw, const float* uh, const float* ud, long long n,
                     float* y, float* lad, int& flag) {
    constexpr int M = nfk::spline_param_count(NB, TAILS);
    constexpr int MP = (M + 7) / 8 * 8;
    constexpr int ND = M - 2 * NB;
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
    const nfk::SplineParams p = nfk::spline_params_of(*desc);
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
