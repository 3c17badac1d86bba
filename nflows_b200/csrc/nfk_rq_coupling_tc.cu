// ONE kernel for the dominant step of PiecewiseRationalQuadraticCouplingTransform (coupling.py:279-293, 549-582 +
// splines/rational_quadratic.py:13-181 in the reference): the final conditioner layer (hidden -> d_t * (3K-1)
// spline parameters, 86 % of the flow's FLOPs) on the tensor cores (wgmma), with the rational-quadratic spline, the scatter
// of the transformed features and the per-row log|det| evaluated by the consumer warpgroups straight from the accumulators.
// The [B, d_t*M] parameter tensor the reference materialises (37.8 GB per layer at B = 2^20) never exists.
//
// Same machinery as nfk_linear_tc.cu (TMA-fed fp16 split-pair operands, partial sums added to running sums in registers);
// what differs:
//   * the packed weight has MP = roundup(M, 8) rows per transformed feature (zero padded), so a column tile of TF * MP <= 128
//     packed rows holds whole features;
//   * at the end of a tile each consumer warpgroup stages its 64 x 128 sums in shared memory and re-reads them one row per
//     thread pair: thread (row, half) owns ALL parameters of FPT = TF / 2 features of its row and evaluates their splines;
//   * a CTA walks the column tiles of one 128-row block consecutively, so every thread keeps the running log|det| of its row
//     in a register and the row is finished (lad_accum updated, deterministically) when the CTA moves on.
#include <stdlib.h>

#include "fused_spline.cuh"

namespace nfk {
namespace tc {

struct FusedParams {
    SplineOut o;            // bias, inputs, outputs, spline (fused_spline.cuh)
    float* lad_accum;       // [n_rows] running log|det| (read-modify-write) or null
    int32_t* flags;
    int64_t n_rows;
    int K;                  // hidden features (GEMM reduction length)
    int num_m_tiles, num_n_tiles;
};

constexpr int FUSED_STAGES = 4;                                 // 4 x 32 KB ring
constexpr int FUSED_STG_OFF = FUSED_STAGES * STAGE_BYTES + 256;   // staged sums: 64 x BN floats per warpgroup (fused_spline.cuh)
constexpr int FUSED_SMEM_BYTES = FUSED_STG_OFF + 2 * 64 * BN * 4 + 1024 /*alignment slack*/;
static_assert(FUSED_SMEM_BYTES <= 232448, "fused kernel shared memory");

template <int NB, bool TAILS>
__global__ void __launch_bounds__(THREADS, 1)
rq_coupling_final_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                         const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                         const FusedParams p) {
    using Cfg = FusedCfg<NB, TAILS>;
    constexpr int TILE = Cfg::TILE;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    const uint32_t bars = smem_base + FUSED_STAGES * STAGE_BYTES;
    Ring ring{smem_base, bars, bars + 8 * FUSED_STAGES, FUSED_STAGES, (uint32_t)STAGE_BYTES};
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_k = (p.K + BK - 1) / BK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < FUSED_STAGES; ++s) { mbar_init(ring.full + 8 * s, 1); mbar_init(ring.empty + 8 * s, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        prefetch_tmap(&map_a_hi); prefetch_tmap(&map_a_lo); prefetch_tmap(&map_w_hi); prefetch_tmap(&map_w_lo);
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");      // registers to the consumer warpgroups
        // ================================================= TMA producer (one elected thread of warp 0)
        if (warp == 0 && elect_one()) {
            for (int mb = blockIdx.x; mb < p.num_m_tiles; mb += gridDim.x)
                for (int n = 0; n < p.num_n_tiles; ++n)
                    for (int ks = 0; ks < num_k; ++ks)
                        produce_slab(ring, &map_a_hi, &map_a_lo, &map_w_hi, &map_w_lo, ks, mb * BM, n * TILE);
        }
        return;
    }
    // ================================================= consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int wg = (warp >> 2) - 1, wi = warp & 3;
    const int t = threadIdx.x - 128 * (1 + wg);
    const int r_loc = t >> 1, fh = t & 1;                   // spline phase: this thread's row of the warpgroup, feature half
    float* stg = reinterpret_cast<float*>(smem_gen + FUSED_STG_OFF) + wg * 64 * BN;
    int flag = 0;
    for (int mb = blockIdx.x; mb < p.num_m_tiles; mb += gridDim.x) {
        const int64_t row = (int64_t)mb * BM + wg * 64 + r_loc;
        const bool row_ok = row < p.n_rows;
        float lad_row = 0.0f;
        for (int n = 0; n < p.num_n_tiles; ++n) {
            const SplineIn<NB, TAILS> in = spline_inputs<NB, TAILS>(p.o, n, row, row_ok, fh);
            float sum[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) sum[i] = 0.0f;
            mma_tile(sum, ring, num_k, DRAIN_SLABS_FUSED, wg, lane);
            wg_sync(wg);                                    // the previous tile's staged sums have been read
            stage_sums<NB, TAILS, BN>(stg, sum, wi, lane);
            wg_sync(wg);
            spline_tile<NB, TAILS>(p.o, stg, r_loc, n, row, row_ok, fh, in, lad_row, flag);
        }
        // ---- finish the row block: lad_accum[row] += the two feature halves' partial sums, fixed order
        const float other = __shfl_xor_sync(0xffffffffu, lad_row, 1);
        if (p.lad_accum && fh == 0 && row_ok) p.lad_accum[row] += lad_row + other;
    }
    if (flag && p.flags) atomicOr(p.flags, flag);
}

template <int NB, bool TAILS>
static int launch_fused(const CUtensorMap& ma_hi, const CUtensorMap& ma_lo, const __half* w_hi, const __half* w_lo, int64_t ldw,
                        FusedParams& p, cudaStream_t st) {
    using Cfg = FusedCfg<NB, TAILS>;
    const int packed_rows = p.o.d_t * Cfg::MP;
    CUtensorMap mw_hi, mw_lo;
    int rc;
    if ((rc = make_map(&mw_hi, w_hi, packed_rows, p.K, ldw, BN))) return rc;
    if ((rc = make_map(&mw_lo, w_lo, packed_rows, p.K, ldw, BN))) return rc;
    p.num_n_tiles = (p.o.d_t + Cfg::TF - 1) / Cfg::TF;
    static DeviceOnce attr_once;
    int attr_dev = 0;
    if (attr_once.pending(&attr_dev)) {
        cudaError_t e = cudaFuncSetAttribute(rq_coupling_final_kernel<NB, TAILS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             FUSED_SMEM_BYTES);
        if (e != cudaSuccess) return fail(NFK_E_CUDA, "cudaFuncSetAttribute(smem=%d): %s", FUSED_SMEM_BYTES, cudaGetErrorString(e));
        attr_once.mark(attr_dev);
    }
    const int grid = p.num_m_tiles < sm_count() ? p.num_m_tiles : sm_count();
    rq_coupling_final_kernel<NB, TAILS><<<grid, THREADS, FUSED_SMEM_BYTES, st>>>(ma_hi, ma_lo, mw_hi, mw_lo, p);
    return check_launch("rq_coupling_final_kernel");
}

}  // namespace tc
}  // namespace nfk

using namespace nfk;

extern "C" int nfk_rq_coupling_final_supported(int32_t num_bins, int32_t linear_tails, int32_t hidden_features, int64_t lda) {
    const bool bins_ok = (num_bins == 8 || num_bins == 10 || num_bins == 4 || num_bins == 16);
    return (bins_ok && hidden_features >= 8 && hidden_features % 8 == 0 && lda % 8 == 0) ? 1 : 0;
}

extern "C" int32_t nfk_rq_coupling_final_padded_params(int32_t num_bins, int32_t linear_tails) {
    const int m = linear_tails ? 3 * num_bins - 1 : 3 * num_bins + 1;
    return (m + 7) / 8 * 8;
}

extern "C" int nfk_rq_coupling_final_f16x3(const NfkSplineDesc* desc, int inverse, const void* a_hi_, const void* a_lo_,
                                          int64_t lda, int32_t a_exp, const void* wp_hi_, const void* wp_lo_, int64_t ldw,
                                          int32_t w_exp, const float* bias_packed, int32_t hidden_features, const float* x,
                                          int64_t ldx, const int32_t* t_cols, int32_t t_col0, int32_t d_t, float* y,
                                          int64_t ldy, void* y_hi, void* y_lo, int64_t lds, int32_t y_exp, float* lad_accum,
                                          int64_t n_rows, int32_t* flags, void* stream) {
    const __half* a_hi = (const __half*)a_hi_; const __half* a_lo = (const __half*)a_lo_;
    const __half* wp_hi = (const __half*)wp_hi_; const __half* wp_lo = (const __half*)wp_lo_;
    tc::FusedParams p;
    int rc = make_spline_params(desc, &p.o.sp);
    if (rc) return rc;
    NFK_REQUIRE(n_rows >= 0 && d_t >= 1 && hidden_features >= 1, "bad sizes");
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(a_hi && a_lo && wp_hi && wp_lo && bias_packed && x, "NULL pointer");
    NFK_REQUIRE((y != nullptr) != (y_hi != nullptr), "give either y (fp32 outputs) or y_hi / y_lo (their fp16 split pair)");
    NFK_REQUIRE((y_hi == nullptr) == (y_lo == nullptr) && y_exp >= -60 && y_exp <= 60, "bad pair output");
    NFK_REQUIRE(t_cols || t_col0 >= 0, "t_cols is NULL and t_col0 is negative");
    NFK_REQUIRE(aligned16(bias_packed), "bias_packed must be 16-byte aligned");
    NFK_REQUIRE(nfk_rq_coupling_final_supported(desc->num_bins, desc->linear_tails, hidden_features, lda) && ldw % 8 == 0,
                "fused coupling kernel does not take num_bins=%d hidden=%d", desc->num_bins, hidden_features);
    NFK_REQUIRE(aligned16(a_hi) && aligned16(a_lo) && aligned16(wp_hi) && aligned16(wp_lo), "operands must be 16-byte aligned");
    NFK_REQUIRE(n_rows < (1ll << 31), "n_rows too large for one launch");
    NFK_REQUIRE(a_exp + w_exp >= -60 && a_exp + w_exp <= 60, "scale exponent out of range");
    p.o.bias = bias_packed; p.o.x = x; p.o.y = y; p.o.y_hi = (__half*)y_hi; p.o.y_lo = (__half*)y_lo; p.o.t_cols = t_cols;
    p.o.t_col0 = t_col0; p.o.out_scale = ldexpf(1.0f, y_exp); p.o.ldx = ldx; p.o.ldy = ldy; p.o.lds = lds; p.o.d_t = d_t;
    p.o.inverse = inverse; p.o.inv_acc_scale = ldexpf(1.0f, -(a_exp + w_exp));
    p.lad_accum = lad_accum; p.flags = flags; p.n_rows = n_rows; p.K = hidden_features;
    p.num_m_tiles = (int)((n_rows + tc::BM - 1) / tc::BM);
    CUtensorMap ma_hi, ma_lo;
    if ((rc = tc::make_map(&ma_hi, a_hi, n_rows, hidden_features, lda, tc::BM))) return rc;
    if ((rc = tc::make_map(&ma_lo, a_lo, n_rows, hidden_features, lda, tc::BM))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const bool tails = desc->linear_tails != 0;
#define NFK_FUSED(NB)                                                                                \
    return tails ? tc::launch_fused<NB, true>(ma_hi, ma_lo, wp_hi, wp_lo, ldw, p, st)                \
                 : tc::launch_fused<NB, false>(ma_hi, ma_lo, wp_hi, wp_lo, ldw, p, st)
    switch (desc->num_bins) {
        case 4: NFK_FUSED(4);
        case 8: NFK_FUSED(8);
        case 10: NFK_FUSED(10);
        case 16: NFK_FUSED(16);
    }
#undef NFK_FUSED
    return fail(NFK_E_UNSUPPORTED, "num_bins=%d has no fused kernel instance", desc->num_bins);
}
