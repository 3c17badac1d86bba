// ONE kernel per PiecewiseRationalQuadraticCouplingTransform step (reference: coupling.py:73-99, 279-293, 549-582 around
// nn/nets/resnet.py:92-100 and splines/rational_quadratic.py:13-181): the WHOLE conditioner -- initial layer, the square
// layers of the residual blocks, the final layer -- on the tensor cores (wgmma), the spline, the scatter of the transformed
// features and the per-row log|det| in the epilogue.  Nothing the conditioner computes goes to global memory but the skip
// tensor of the residual blocks:
//
//   * a CTA owns a 128-row tile from the first layer to the spline.  The activation of the tile lives in shared memory as the
//     K-major fp16 (hi, lo) split pair the NEXT layer multiplies ("R": H / 32 K-slabs x [hi 8 KB | lo 8 KB], up to 128 KB,
//     written by the consumer warpgroups in the SWIZZLE_64B placement the wgmma descriptors read); only weights stream, by TMA;
//   * in the trunk, consumer warpgroup w multiplies and writes rows [64 w, 64 w + 64) of R only, so between the layers of a
//     tile each warpgroup synchronises with itself alone;
//   * a layer wider than 128 columns runs as two 128-column chunks: the first chunk's output pair waits in a per-warpgroup
//     scratch area ("S", 32 KB each) until the second chunk's MMAs have read R, then both are written into R;
//   * the final layer walks the column tiles of the packed weight (fused_spline.cuh: FusedCfg; MMAs of N = TILE columns, the
//     tile's packed rows and no more) against the SAME resident operand, in ping-pong: warpgroup n % 2 takes column tile n for
//     all 128 rows, so one warpgroup's MMAs run while the other stages its sums in S (two 64-row passes) and evaluates the
//     spline (fused_spline.cuh: spline_tile).  The tile's packed bias is copied into shared memory (cp.async) before its MMAs
//     are waited for.  With a single column tile (the autoregressive inverse) there is nothing to overlap, and both
//     warpgroups take it, each for its own 64 rows;
//   * the residual-block skip tensor goes through a per-CTA fp32 scratch (one 128 x H tile per CTA, L2-resident, every thread
//     reads back exactly what it wrote).
//
// The instances with NB = AFFINE_NB (fused_spline.cuh) run the masked autoregressive transform's affine map instead of the
// spline in the same place (nfk_affine_ar_step_f16x3): the final layer is MADE's, 2 rows per feature, TILE = 128.
//
// Arithmetic is that of nfk_linear_tc.cu / nfk_rq_coupling_tc.cu: fp16 split pairs with power-of-two scales, three f16 MMAs
// per K-step, partial sums of 4 (trunk) K-slabs added to running sums with round-to-nearest; the final layer's K (<= 8 slabs) is
// one partial sum.
//
// Shared memory (dynamic, 1024-aligned):
//   [0, 128 KB)         R; during the initial layer (R is dead until its epilogue) 4 stages x 32 KB [A hi | A lo | W hi | W lo]
//   [128 KB, 192 KB)    S: in the trunk, per consumer warpgroup 32 KB for the first chunk's output pair.  In the final layer
//                       the staged sums, 64 rows x FusedCfg::LD floats per warpgroup (24 KB at TILE = 96, 32 KB otherwise);
//                       in the ping-pong warpgroup 1's follow warpgroup 0's, with a single column tile each warpgroup
//                       stages in its own 32 KB
//   [192 KB, 224 KB)    weight ring of the square layers: 2 stages x 16 KB [W hi | W lo].  The final layer uses it too at
//                       TILE = 112 and 128 and with a single column tile (a slab fills TILE rows of each half)
//   [176 KB, 224 KB)    TILE = 96 with two or more column tiles: the final layer's own ring, 4 stages x 12 KB [W hi | W lo at
//                       +6 KB], over the top 16 KB of S the staging leaves free and the trunk's ring (StepFinal below)
//   then the barriers, warpgroup 1's per-row log|det| shares (512 bytes) and per consumer warpgroup the packed bias of its
//   column tile (up to BN floats).
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "fused_spline.cuh"

namespace nfk {
namespace tc {

constexpr int STEP_MAX_LAYERS = 9;                                   // initial layer + up to 8 square layers
static_assert(STEP_MAX_LAYERS == NFK_STEP_MAX_LAYERS, "include/nfk.h: NfkStepRowTerms");
constexpr int STEP_MAX_HIDDEN = 256;
constexpr int STEP_DRAIN_TRUNK = 4;                                  // K-slabs per partial sum: trunk layers
constexpr int STEP_DRAIN_FINAL = 8;                                  // ... final layer (spline logits): K = 256 at once
constexpr int STEP_SLAB_BYTES = 2 * A_BYTES;                         // one K-slab of R: hi | lo
constexpr int STEP_R_BYTES = (STEP_MAX_HIDDEN / BK) * STEP_SLAB_BYTES;   // 128 KB
constexpr int STEP_G0_STAGES = STEP_R_BYTES / STAGE_BYTES;           // 4
constexpr int STEP_S_OFF = STEP_R_BYTES;
constexpr int STEP_S_WG_BYTES = 32768;                               // per consumer warpgroup
constexpr int STEP_W_OFF = STEP_S_OFF + 2 * STEP_S_WG_BYTES;
constexpr int STEP_W_STAGES = 2;
constexpr int STEP_W_STAGE_BYTES = 2 * B_BYTES;
constexpr int STEP_BAR_OFF = STEP_W_OFF + STEP_W_STAGES * STEP_W_STAGE_BYTES;
constexpr int STEP_LAD_OFF = STEP_BAR_OFF + 256;                    // warpgroup 1's per-row log|det| shares: 128 floats
constexpr int STEP_BIAS_OFF = STEP_LAD_OFF + 512;                   // per consumer warpgroup BN floats: its tile's packed bias
constexpr int STEP_SMEM_BYTES = STEP_BIAS_OFF + 2 * BN * 4 + 1024 /*alignment slack*/;
static_assert(64 * BN * 4 <= STEP_S_WG_BYTES && 4 * 2 * 64 * 64 <= STEP_S_WG_BYTES, "S");
static_assert(STEP_SMEM_BYTES <= 232448, "coupling-step kernel shared memory");
static_assert(STEP_MAX_HIDDEN / BK <= STEP_DRAIN_FINAL, "the final layer drains once (mma_final)");

// The final layer's weight ring of the ping-pong.  Staged at a row stride of LD floats, the two warpgroups' sums leave the top
// of S free; together with the trunk's ring that makes STAGES slots of TILE-row [W hi | W lo] slabs: 4 at TILE = 96, 2 at
// TILE = 112 and 128, where the final layer keeps the trunk's ring (and its bytes) instead.
template <int NB, bool TAILS>
struct StepFinal {
    static constexpr int TILE = FusedCfg<NB, TAILS>::TILE, LD = FusedCfg<NB, TAILS>::LD;
    static constexpr int STG_BYTES = 64 * LD * 4;                   // one warpgroup's staged 64-row pass
    static constexpr int RING_OFF = STEP_S_OFF + 2 * STG_BYTES;
    static constexpr int LO_OFF = TILE * ROW_BYTES;                  // W lo within a slot
    static constexpr int STAGE_BYTES = 2 * LO_OFF;
    static constexpr int STAGES = (STEP_BAR_OFF - RING_OFF) / STAGE_BYTES;
    static constexpr bool OWN_RING = STAGES > STEP_W_STAGES;
    static_assert(STG_BYTES <= STEP_S_WG_BYTES, "S");
    // SWIZZLE_64B: TMA boxes and wgmma descriptors agree on slots and W lo halves that start at multiples of 512 bytes
    static_assert(RING_OFF % 512 == 0 && LO_OFF % 512 == 0 && STAGE_BYTES % 512 == 0, "final ring alignment");
    static_assert(!OWN_RING || (STAGES == 4 && RING_OFF >= STEP_S_OFF + STEP_S_WG_BYTES), "final ring");
    static_assert(112 + 2 * 8 * STAGES <= STEP_LAD_OFF - STEP_BAR_OFF, "its mbarriers follow bar_sfree");
};

#ifdef NFK_STEP_CLOCKS
// Phase clocks (scripts/step_phases.py): clock64 stamps by thread 0 of each consumer warpgroup of CTAs [0, CLK_CTAS), on their
// row tiles of rounds 1 .. CLK_ROUNDS (round 0 warms up).  Per (CTA, round): trunk start / end of each warpgroup, then per
// column tile n < CLK_TILES (its owner's stamps): before the turn wait, first slab landed, last slab landed, MMAs retired, and
// per 64-row pass: sums staged, spline done.  Not in the shipped library.
constexpr int CLK_CTAS = 8, CLK_ROUNDS = 3, CLK_TILES = 128, CLK_TILE_STAMPS = 8;
constexpr int CLK_REC = 4 + CLK_TILES * CLK_TILE_STAMPS;
__device__ long long g_step_clocks[CLK_CTAS * CLK_ROUNDS * CLK_REC];
#define NFK_CLK(ptr, i) \
    do {                \
        if (ptr) (ptr)[i] = clock64(); \
    } while (0)
__device__ __forceinline__ long long* step_clock_record(int u, int t) {
    const int round = (u - (int)blockIdx.x) / (int)gridDim.x;
    if (t != 0 || blockIdx.x >= CLK_CTAS || round < 1 || round > CLK_ROUNDS) return nullptr;
    return g_step_clocks + ((int)blockIdx.x * CLK_ROUNDS + round - 1) * CLK_REC;
}
#define NFK_CLK_RECORD(u, t) step_clock_record(u, t)
#define NFK_CLK_TILE(rec, n) ((rec) && (n) < CLK_TILES ? (rec) + 4 + (n) * CLK_TILE_STAMPS : nullptr)
#else
#define NFK_CLK(ptr, i) \
    do {                \
    } while (0)
#define NFK_CLK_RECORD(u, t) ((long long*)nullptr)
#define NFK_CLK_TILE(rec, n) ((long long*)nullptr)
#endif

// layer_flags bits (include/nfk.h: NfkCouplingStep)
constexpr int SL_RELU_OUT = 1;     // relu on (acc + bias)
constexpr int SL_ADD_SKIP = 2;     // + the saved skip tensor (never combined with SL_RELU_OUT)
constexpr int SL_SAVE_SKIP = 4;    // the fp32 result is the skip tensor of a later layer
constexpr int SL_SPLIT_RELU = 8;   // the consumer of this layer's output applies relu to its input
constexpr int SL_ACT_SHIFT = 8;    // bits [8, 12): the activation (NFK_ACT_*) of bits 1 and 8; 0 reads as relu
constexpr int SL_ACT_MASK = 15;

__host__ __device__ __forceinline__ int layer_act(int lf) {
    const int a = (lf >> SL_ACT_SHIFT) & SL_ACT_MASK;
    return a ? a : NFK_ACT_RELU;
}

template <int ACT>
__device__ __forceinline__ void act_frag(float (&v)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) v[i] = nfk_act(ACT, v[i]);
}

// The activation of a layer on a thread's 64 accumulator values, chosen once for the fragment (relu: fmaxf, as it always was).
__device__ __forceinline__ void act_fragment(int act, float (&v)[64]) {
    switch (act) {
        case NFK_ACT_RELU: act_frag<NFK_ACT_RELU>(v); break;
        case NFK_ACT_TANH: act_frag<NFK_ACT_TANH>(v); break;
        case NFK_ACT_ELU: act_frag<NFK_ACT_ELU>(v); break;
        case NFK_ACT_LEAKY_RELU: act_frag<NFK_ACT_LEAKY_RELU>(v); break;
        case NFK_ACT_GELU: act_frag<NFK_ACT_GELU>(v); break;
        case NFK_ACT_SILU: act_frag<NFK_ACT_SILU>(v); break;
    }
}

struct StepParams {
    // ---- conditioner trunk
    const float* bias_trunk;      // [num_layers * H]: initial layer, then the square layers
    float* skip_buf;              // [gridDim.x][128][H] scratch
    int H, K0, num_layers;        // num_layers = 1 + number of square layers
    int layer_flags[STEP_MAX_LAYERS];
    float acc_scale[STEP_MAX_LAYERS], inv_acc_scale[STEP_MAX_LAYERS];
    float act_scale;              // 2^e_act: exponent of every hidden activation pair
    __half* h_hi;                 // non-null: stop after the trunk, its output pair goes here [n_rows, ldh]
    __half* h_lo;
    int64_t ldh;
    // ---- final layer + spline
    SplineOut o;
    float* lad_accum;
    int32_t* flags;
    int64_t n_rows;
    int num_m_tiles, num_n_tiles;
};

// Per-row additive terms of the trunk layers (include/nfk.h: NfkStepRowTerms): layer l computes post(acc + bias + add[l][row, col])
// (+ skip).  A separate parameter type of the TERMS instances only, so the instances without terms keep their parameter block.
struct StepTermParams : StepParams {
    const float* add[STEP_MAX_LAYERS];   // fp32 [n_rows, ld_add[l]] or null
    int64_t ld_add[STEP_MAX_LAYERS];
};

// The mixture instances' parameters (always with the terms: p.add[l] null means none).
struct StepMogParams : StepTermParams {
    MogOut mog;
};

template <int NB, bool TERMS>
using StepParamsOf = typename std::conditional<FusedCfg<NB, false>::MOG, StepMogParams,
                                               typename std::conditional<TERMS, StepTermParams, StepParams>::type>::type;

// The fp16 split pair of (x0, x1) * scale for columns (col, col + 1) of row r of a K-major SWIZZLE_64B operand: K-slab
// col / 32 at base + (col / 32) * slab_stride, hi part first, lo part lo_off bytes after it, 64-byte rows.
__device__ __forceinline__ void put_pair(uint8_t* base, int slab_stride, int lo_off, int r, int col, float x0, float x1, float scale,
                                         float& amax) {
    x0 *= scale; x1 *= scale;
    amax = fmaxf(amax, fmaxf(fabsf(x0), fabsf(x1)));
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    const int k = col & 31;
    uint8_t* q = base + (col >> 5) * slab_stride + r * 64 + (((k >> 3) ^ ((r >> 1) & 3)) << 4) + (k & 7) * 2;
    *reinterpret_cast<__half2*>(q) = h;
    *reinterpret_cast<__half2*>(q + lo_off) = l;
}

__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 3, 256;" ::: "memory"); }
constexpr int STEP_BAR_TURN = 4;   // + w: warpgroup w may wait on its next final-layer tile (ids 4, 5)
constexpr int STEP_BAR_LAD = 6;    // warpgroup 1's log|det| shares are in shared memory

// Final layer: one column tile of N packed rows (FusedCfg::TILE) against the resident operand, MH 64-row halves of it from
// a_res on.  MH = 2: the ping-pong, one warpgroup takes the tile for all 128 rows and is the only consumer of its slabs (each
// warp arrives twice on the `empty` barriers, which count 8).  MH = 1: both warpgroups take the tile, each for its own rows.
// The arithmetic of mma_tile with a single partial sum over the whole K (H <= 256 = STEP_DRAIN_FINAL slabs), so the
// accumulators are the sums.  turn >= 0: signal that named barrier once the last slab has landed.  W lo lies lo_off bytes
// after W hi in a slot.  clk (phase-clock builds only): stamps 1 - 3 of the tile.
template <int N, int MH>
__device__ __forceinline__ void mma_final(float (&acc)[MH][N / 2], Ring& r, int num_k, uint32_t a_res, int lane, int turn,
                                          uint32_t lo_off, [[maybe_unused]] long long* clk) {
    int prev = -1;
    for (int j = 0; j < num_k; ++j) {
        mbar_wait(r.full + 8 * r.stage, r.phase);
        if (j == 0) NFK_CLK(clk, 1);
        if (j == num_k - 1) NFK_CLK(clk, 2);
        if (turn >= 0 && j == num_k - 1) {
            __threadfence_block();
            pair_arrive(turn);
        }
        const uint32_t sw = r.base + r.stage * r.stage_bytes;
        const uint64_t w_hi = make_smem_desc(sw), w_lo = make_smem_desc(sw + lo_off);
        wgmma_fence();
#pragma unroll
        for (int m = 0; m < MH; ++m) {
            const uint32_t sa = a_res + (uint32_t)j * STEP_SLAB_BYTES + m * (A_BYTES / 2);
            const uint64_t a_hi = make_smem_desc(sa), a_lo = make_smem_desc(sa + A_BYTES);
#pragma unroll
            for (int kk = 0; kk < BK / 16; ++kk) {
                const uint64_t adv = (uint64_t)(kk * 2);
                wgmma_f16<N>(acc[m], a_lo + adv, w_hi + adv, (j | kk) != 0);
                wgmma_f16<N>(acc[m], a_hi + adv, w_lo + adv, 1);
            }
#pragma unroll
            for (int kk = 0; kk < BK / 16; ++kk) {
                const uint64_t adv = (uint64_t)(kk * 2);
                wgmma_f16<N>(acc[m], a_hi + adv, w_hi + adv, 1);
            }
        }
        wgmma_commit();
        if (prev >= 0) {
            wgmma_wait<1>();
            __syncwarp();
            if (lane == 0) mbar_arrive(r.empty + 8 * prev, MH);
        }
        prev = r.stage;
        r.advance();
    }
    wgmma_wait<0>();
    NFK_CLK(clk, 3);
    __syncwarp();
    if (lane == 0) mbar_arrive(r.empty + 8 * prev, MH);
}

// ACT: the instance for layer flags with an activation field (any activation); the instances without it apply relu only, as
// they always did, so the relu path keeps its code and registers.
template <int NB, bool TAILS, bool TERMS, bool ACT>
__global__ void __launch_bounds__(THREADS, 1)
rq_coupling_step_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                        const __grid_constant__ CUtensorMap map_w0_hi, const __grid_constant__ CUtensorMap map_w0_lo,
                        const __grid_constant__ CUtensorMap map_wt_hi, const __grid_constant__ CUtensorMap map_wt_lo,
                        const __grid_constant__ CUtensorMap map_wf_hi, const __grid_constant__ CUtensorMap map_wf_lo,
                        const StepParamsOf<NB, TERMS> p) {
    using F = StepFinal<NB, TAILS>;
    constexpr int TILE = F::TILE;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    const uint32_t bars = smem_base + STEP_BAR_OFF;
    Ring ring0{smem_base, bars, bars + 8 * STEP_G0_STAGES, STEP_G0_STAGES, (uint32_t)STAGE_BYTES};
    Ring ring1{smem_base + STEP_W_OFF, bars + 64, bars + 64 + 8 * STEP_W_STAGES, STEP_W_STAGES, (uint32_t)STEP_W_STAGE_BYTES};
    // the ping-pong's final-layer ring: its own slots and barriers where StepFinal makes room for them, else the trunk's ring
    Ring ring_own{smem_base + F::RING_OFF, bars + 112, bars + 112 + 8 * F::STAGES, F::STAGES, (uint32_t)F::STAGE_BYTES};
    Ring& ringf = F::OWN_RING ? ring_own : ring1;
    constexpr uint32_t lo_f = F::OWN_RING ? F::LO_OFF : B_BYTES;
    const uint32_t bar_rfree = bars + 96;          // the consumers' last MMAs of a tile have read R
    const uint32_t bar_sfree = bars + 104;         // OWN_RING: both consumer warpgroups are past their last trunk use of S
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int H = p.H;
    const int num_k0 = (p.K0 + BK - 1) / BK, num_kh = H / BK;
    const int nch = (H + BN - 1) / BN;               // 128-column chunks of a trunk layer
    const bool trunk_only = p.h_hi != nullptr;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STEP_G0_STAGES; ++s) { mbar_init(ring0.full + 8 * s, 1); mbar_init(ring0.empty + 8 * s, 8); }
        for (int s = 0; s < STEP_W_STAGES; ++s) { mbar_init(ring1.full + 8 * s, 1); mbar_init(ring1.empty + 8 * s, 8); }
        mbar_init(bar_rfree, 8);
        if constexpr (F::OWN_RING) {
            for (int s = 0; s < F::STAGES; ++s) { mbar_init(ring_own.full + 8 * s, 1); mbar_init(ring_own.empty + 8 * s, 8); }
            mbar_init(bar_sfree, 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        prefetch_tmap(&map_a_hi); prefetch_tmap(&map_a_lo); prefetch_tmap(&map_w0_hi); prefetch_tmap(&map_w0_lo);
        prefetch_tmap(&map_wt_hi); prefetch_tmap(&map_wt_lo); prefetch_tmap(&map_wf_hi); prefetch_tmap(&map_wf_lo);
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");      // registers to the consumer warpgroups
        // ================================================= TMA producer (one elected thread of warp 0)
        if (warp == 0 && elect_one()) {
            uint32_t rphase = 0, sphase = 0;
            for (int u = blockIdx.x; u < p.num_m_tiles; u += gridDim.x) {
                if (u != (int)blockIdx.x) { mbar_wait(bar_rfree, rphase); rphase ^= 1; }   // the initial-layer stages lie over R
                for (int c = 0; c < nch; ++c)
                    for (int ks = 0; ks < num_k0; ++ks) produce_slab(ring0, &map_a_hi, &map_a_lo, &map_w0_hi, &map_w0_lo, ks, u * BM, c * BN);
                for (int l = 1; l < p.num_layers; ++l)
                    for (int c = 0; c < nch; ++c)
                        for (int ks = 0; ks < num_kh; ++ks) produce_w_slab(ring1, &map_wt_hi, &map_wt_lo, ks, (l - 1) * H + c * BN);
                if (trunk_only) continue;
                if (F::OWN_RING && p.num_n_tiles > 1) {
                    // The final ring lies over the top of S and over the trunk's ring: wait until both consumer warpgroups are
                    // past their last trunk use of S and the trunk ring's last slabs have been read.  The next tile's initial
                    // layer (over R) and its trunk slabs wait for bar_rfree, which follows the last final-layer MMAs.
                    mbar_wait(bar_sfree, sphase);
                    sphase ^= 1;
                    Ring w = ring1;
                    for (int s = 0; s < STEP_W_STAGES; ++s) {
                        mbar_wait(w.empty + 8 * w.stage, w.phase ^ 1);
                        w.advance();
                    }
                    for (int n = 0; n < p.num_n_tiles; ++n)
                        for (int ks = 0; ks < num_kh; ++ks) produce_w_slab(ring_own, &map_wf_hi, &map_wf_lo, ks, n * TILE, TILE, F::LO_OFF);
                } else {
                    for (int n = 0; n < p.num_n_tiles; ++n)
                        for (int ks = 0; ks < num_kh; ++ks) produce_w_slab(ring1, &map_wf_hi, &map_wf_lo, ks, n * TILE, TILE);
                }
            }
        }
        return;
    }
    // ================================================= consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int wg = (warp >> 2) - 1, wi = warp & 3, q = lane & 3;
    const int t = threadIdx.x - 128 * (1 + wg);
    const int r_loc = t >> 1, fh = t & 1;            // spline phase: this thread's row of the warpgroup, feature half
    uint8_t* R = smem_gen;
    uint8_t* S = smem_gen + STEP_S_OFF + wg * STEP_S_WG_BYTES;
    float* stg = reinterpret_cast<float*>(S);
    float* const bias_wg = reinterpret_cast<float*>(smem_gen + STEP_BIAS_OFF) + wg * BN;   // the packed bias of this warpgroup's tile
    float* skip = p.skip_buf + (size_t)blockIdx.x * BM * H;
    int flag = 0;
    for (int u = blockIdx.x; u < p.num_m_tiles; u += gridDim.x) {
        const int64_t m0 = (int64_t)u * BM;
        int rt[2];                                   // rows (within the tile) of this thread's accumulator fragments
        rt[0] = wg * 64 + wi * 16 + (lane >> 2);
        rt[1] = rt[0] + 8;
        [[maybe_unused]] long long* const clk = NFK_CLK_RECORD(u, t);
        NFK_CLK(clk, 2 * wg);
        // ------------------------------------------------ conditioner trunk: layer l's epilogue writes layer l+1's operand into R
        for (int l = 0; l < p.num_layers; ++l) {
            const int lf = p.layer_flags[l];
            [[maybe_unused]] const int act = layer_act(lf);
            const bool to_global = trunk_only && l == p.num_layers - 1;
            const float as = p.acc_scale[l], ias = p.inv_acc_scale[l];
            float amax = 0.0f;
            for (int c = 0; c < nch; ++c) {
                const int cb = c * BN + 2 * q;       // column of sum[4 j + 2 h + e] is cb + 8 j + e
                float sum[64];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = cb + 8 * j;
                    [[maybe_unused]] float2 tv[2] = {make_float2(0.0f, 0.0f), make_float2(0.0f, 0.0f)};
                    if constexpr (TERMS) {           // the row term of (row, col), (row, col + 1); rows past n_rows are not read
                        const float* ta = p.add[l];
                        if (ta != nullptr && col < H) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const int64_t row = m0 + rt[h];
                                if (row < p.n_rows) tv[h] = __ldg(reinterpret_cast<const float2*>(ta + row * p.ld_add[l] + col));
                            }
                        }
                    }
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float b = col < H ? __ldg(p.bias_trunk + l * H + col + e) * as : 0.0f;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            float sk = ((lf & SL_ADD_SKIP) && col < H) ? skip[rt[h] * H + col + e] : 0.0f;
                            if constexpr (TERMS) sk += e ? tv[h].y : tv[h].x;
                            sum[4 * j + 2 * h + e] = fmaf(sk, as, b);
                        }
                    }
                }
                if (l == 0) mma_tile(sum, ring0, num_k0, STEP_DRAIN_TRUNK, wg, lane);
                else mma_tile(sum, ring1, num_kh, STEP_DRAIN_TRUNK, wg, lane, smem_base);
#pragma unroll
                for (int i = 0; i < 64; ++i) {
                    float x = sum[i] * ias;
                    if (!ACT && (lf & SL_RELU_OUT)) x = fmaxf(x, 0.0f);
                    sum[i] = x;
                }
                if (ACT && (lf & SL_RELU_OUT)) act_fragment(act, sum);
                if (lf & SL_SAVE_SKIP) {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            if (cb + 8 * j < H)
                                *reinterpret_cast<float2*>(skip + rt[h] * H + cb + 8 * j) = make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
                }
                if (lf & SL_SPLIT_RELU) {
                    if constexpr (ACT) {
                        act_fragment(act, sum);
                    } else {
#pragma unroll
                        for (int i = 0; i < 64; ++i) sum[i] = fmaxf(sum[i], 0.0f);
                    }
                }
                if (to_global) {                     // trunk output pair straight to global memory
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int64_t row = m0 + rt[h];
                        if (row >= p.n_rows) continue;
                        float am = 0.0f;
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int col = cb + 8 * j;
                            if (col >= H) continue;
                            const float x0 = sum[4 * j + 2 * h] * p.act_scale, x1 = sum[4 * j + 2 * h + 1] * p.act_scale;
                            am = fmaxf(am, fmaxf(fabsf(x0), fabsf(x1)));
                            const __half2 hh = __floats2half2_rn(x0, x1);
                            const float2 hf = __half22float2(hh);
                            *reinterpret_cast<__half2*>(p.h_hi + row * p.ldh + col) = hh;
                            *reinterpret_cast<__half2*>(p.h_lo + row * p.ldh + col) = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
                        }
                        if (!(am <= 65000.0f)) flag |= 4;
                    }
                    continue;
                }
                const bool into_r = c == nch - 1;
                if (into_r) {
                    // every MMA that reads R is done: this warpgroup's (mma_tile waited for them) and, in the initial layer, whose
                    // stages lie over R, the other warpgroup's as well
                    if (l == 0) consumers_sync();
                } else {
                    wg_sync(wg);                     // S is free: the previous tile's staged sums have been read
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float am = 0.0f;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int cc = 8 * j + 2 * q;    // column within the chunk
                        if (c * BN + cc >= H) continue;
                        if (into_r)
                            put_pair(R, STEP_SLAB_BYTES, A_BYTES, rt[h], c * BN + cc, sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1], p.act_scale, am);
                        else
                            put_pair(S, 2 * A_BYTES / 2, A_BYTES / 2, rt[h] - wg * 64, cc, sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1],
                                     p.act_scale, am);
                    }
                    if (m0 + rt[h] < p.n_rows) amax = fmaxf(amax, am);
                }
                if (into_r && nch > 1) {
                    // the first chunk's pair from S into R: K-slab s, hi / lo part, this warpgroup's 64 rows = 4 KB each
                    wg_sync(wg);
                    for (int i = t; i < 4 * 2 * 256; i += 128) {
                        const int part = i >> 8, k = i & 255;   // part = 2 s + lo
                        const uint4 v = reinterpret_cast<const uint4*>(S + part * 4096)[k];
                        reinterpret_cast<uint4*>(R + (part >> 1) * STEP_SLAB_BYTES + (part & 1) * A_BYTES + wg * 4096)[k] = v;
                    }
                }
            }
            if (!(amax <= 65000.0f)) flag |= 4;
            if (!to_global) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> wgmma reads
                wg_sync(wg);
            }
        }
        NFK_CLK(clk, 2 * wg + 1);
        if (trunk_only) {
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_rfree);
            continue;
        }
        // ------------------------------------------------ final layer + spline: the column tiles of this row block
        if (p.num_n_tiles == 1) {
            // a single column tile (the autoregressive inverse) leaves nothing to overlap: both warpgroups share it by rows
            const int64_t srow = m0 + wg * 64 + r_loc;
            const bool row_ok = srow < p.n_rows;
            const SplineIn<NB, TAILS> in = spline_inputs<NB, TAILS>(p.o, 0, srow, row_ok, fh);
            bias_tile_async<NB, TAILS>(bias_wg, p.o, 0, t);   // the last reads of the buffer precede the trunk's barriers
            float acc[1][TILE / 2] = {};        // defined before the MMAs, which read it: no false live range
            mma_final<TILE, 1>(acc, ring1, num_kh, smem_base + wg * (A_BYTES / 2), lane, -1, B_BYTES, nullptr);
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_rfree);
            stage_sums<NB, TAILS, TILE, F::LD>(stg, acc[0], wi, lane);   // S is free: the trunk's last wg_sync follows its last read
            cp_async_wait_all();
            wg_sync(wg);
            float lad_row = 0.0f;
            if constexpr (FusedCfg<NB, TAILS>::MOG)
                mog_tile<NB, TAILS, F::LD>(p.o, p.mog, stg, r_loc, 0, srow, row_ok, fh, in, lad_row, bias_wg);
            else
                spline_tile<NB, TAILS, F::LD, true>(p.o, stg, r_loc, 0, srow, row_ok, fh, in, lad_row, flag, bias_wg);
            const float other = __shfl_xor_sync(0xffffffffu, lad_row, 1);
            if (p.lad_accum && fh == 0 && row_ok) p.lad_accum[srow] += lad_row + other;
            continue;
        }
        // Ping-pong: warpgroup n % 2 owns column tile n for all 128 rows, so one warpgroup's MMAs run while the other evaluates
        // its spline.  The producer's order is unchanged: the ring hands the slabs out in the order the warpgroups take them.
        consumers_sync();                            // R holds all 128 rows: both warpgroups' last trunk epilogues are written
        if constexpr (F::OWN_RING)
            if (t == 0 && wg == 0) mbar_arrive(bar_sfree);   // ... and S is no longer the trunk's: the final ring may fill
        float* const stg_pp = reinterpret_cast<float*>(smem_gen + STEP_S_OFF + wg * F::STG_BYTES);
        const int nt = p.num_n_tiles;
        int64_t srow[2];
        bool row_ok[2];
        float lad[2] = {0.0f, 0.0f};                 // log|det| shares of rows r_loc and 64 + r_loc over this warpgroup's tiles
#pragma unroll
        for (int m = 0; m < 2; ++m) {
            srow[m] = m0 + 64 * m + r_loc;
            row_ok[m] = srow[m] < p.n_rows;
        }
        for (int n = 0; n < nt; ++n) {
            if ((n & 1) != wg) {                     // the other warpgroup's tile: step the ring past its slabs
                for (int ks = 0; ks < num_kh; ++ks) ringf.advance();
                continue;
            }
            [[maybe_unused]] long long* const clk_t = NFK_CLK_TILE(clk, n);
            SplineIn<NB, TAILS> in[2];
#pragma unroll
            for (int m = 0; m < 2; ++m) in[m] = spline_inputs<NB, TAILS>(p.o, n, srow[m], row_ok[m], fh);
            NFK_CLK(clk_t, 0);
            // A slot's `full` barrier is waited on by parity, which tells only two consecutive fills apart: waiting on fill f of
            // a slot is safe once fill f - 1 has landed (fill f + 1 cannot start before this warpgroup releases fill f).  With 4
            // slots and up to 8 slabs a tile fills a slot twice; the fill before one of tile n's slabs is then an earlier slab
            // of tile n (waited on in order) or a slab of an earlier tile.  So tile n - 1's slabs must all have landed before
            // this warpgroup waits on tile n's: their owner says so once it has seen the last of them.  Tile n - 2 was this
            // warpgroup's own, and the tiles before it were covered by the same handshake.
            if (n > 0) pair_wait(STEP_BAR_TURN + wg);
            // every thread of this warpgroup is past pair_wait (or, at n < 2, past the trunk's barriers): the previous
            // tile's spline has read the bias buffer
            bias_tile_async<NB, TAILS>(bias_wg, p.o, n, t);
            float acc[2][TILE / 2] = {};
            mma_final<TILE, 2>(acc, ringf, num_kh, smem_base, lane, n + 1 < nt ? STEP_BAR_TURN + (wg ^ 1) : -1, lo_f, clk_t);
            if (n + 2 >= nt) {                       // this warpgroup's last MMAs on R
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_rfree);
            }
#pragma unroll
            for (int m = 0; m < 2; ++m) {            // two 64-row passes through this warpgroup's S
                wg_sync(wg);                         // S is free: the previous pass has been read
                stage_sums<NB, TAILS, TILE, F::LD>(stg_pp, acc[m], wi, lane);
                if (m == 0) cp_async_wait_all();
                wg_sync(wg);
                NFK_CLK(clk_t, 4 + 2 * m);
                if constexpr (FusedCfg<NB, TAILS>::MOG)
                    mog_tile<NB, TAILS, F::LD>(p.o, p.mog, stg_pp, r_loc, n, srow[m], row_ok[m], fh, in[m], lad[m], bias_wg);
                else
                    spline_tile<NB, TAILS, F::LD, true>(p.o, stg_pp, r_loc, n, srow[m], row_ok[m], fh, in[m], lad[m], flag, bias_wg);
                NFK_CLK(clk_t, 5 + 2 * m);
            }
        }
        // ---- finish the row block: lad_accum[row] += (warpgroup 0's share + warpgroup 1's share), each the sum of its two
        // feature halves -- a fixed order
        float* lad_x = reinterpret_cast<float*>(smem_gen + STEP_LAD_OFF);
#pragma unroll
        for (int m = 0; m < 2; ++m) lad[m] += __shfl_xor_sync(0xffffffffu, lad[m], 1);
        if (wg == 1) {
            if (fh == 0) {
                lad_x[r_loc] = lad[0];
                lad_x[64 + r_loc] = lad[1];
            }
            __threadfence_block();
            pair_arrive(STEP_BAR_LAD);               // read by warpgroup 0 before this warpgroup's next write (after the trunk's
        } else {                                     // consumers_sync of the next row block)
            pair_wait(STEP_BAR_LAD);
            if (p.lad_accum && fh == 0)
#pragma unroll
                for (int m = 0; m < 2; ++m)
                    if (row_ok[m]) p.lad_accum[srow[m]] += lad[m] + lad_x[64 * m + r_loc];
        }
    }
    if (flag && p.flags) atomicOr(p.flags, flag);
}

template <int NB, bool TAILS, bool TERMS, bool ACT>
static int start_step(const CUtensorMap (&m)[8], int grid, StepParamsOf<NB, TERMS>& p, cudaStream_t st) {
    static DeviceOnce attr_once;
    int attr_dev = 0;
    if (attr_once.pending(&attr_dev)) {
        cudaError_t e = cudaFuncSetAttribute(rq_coupling_step_kernel<NB, TAILS, TERMS, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             STEP_SMEM_BYTES);
        if (e != cudaSuccess) return fail(NFK_E_CUDA, "cudaFuncSetAttribute(smem=%d): %s", STEP_SMEM_BYTES, cudaGetErrorString(e));
        attr_once.mark(attr_dev);
    }
    rq_coupling_step_kernel<NB, TAILS, TERMS, ACT><<<grid, THREADS, STEP_SMEM_BYTES, st>>>(m[0], m[1], m[2], m[3], m[4], m[5], m[6],
                                                                                         m[7], p);
    return check_launch("rq_coupling_step_kernel");
}

template <int NB, bool TAILS, bool TERMS>
static int launch_step(const NfkCouplingStep* d, StepParamsOf<NB, TERMS>& p, cudaStream_t st) {
    using Cfg = FusedCfg<NB, TAILS>;
    const int H = p.H, L = p.num_layers - 1;
    CUtensorMap ma_hi, ma_lo, mw0_hi, mw0_lo, mwt_hi, mwt_lo, mwf_hi, mwf_lo;
    int rc;
    if ((rc = make_map(&ma_hi, (const __half*)d->a_hi, p.n_rows, p.K0, d->lda, BM))) return rc;
    if ((rc = make_map(&ma_lo, (const __half*)d->a_lo, p.n_rows, p.K0, d->lda, BM))) return rc;
    if ((rc = make_map(&mw0_hi, (const __half*)d->w0_hi, H, p.K0, d->ldw0, BN))) return rc;
    if ((rc = make_map(&mw0_lo, (const __half*)d->w0_lo, H, p.K0, d->ldw0, BN))) return rc;
    mwt_hi = mw0_hi; mwt_lo = mw0_lo;                          // placeholders when there is no square layer
    if (L > 0) {
        if ((rc = make_map(&mwt_hi, (const __half*)d->wt_hi, (int64_t)L * H, H, d->ldwt, BN))) return rc;
        if ((rc = make_map(&mwt_lo, (const __half*)d->wt_lo, (int64_t)L * H, H, d->ldwt, BN))) return rc;
    }
    mwf_hi = mw0_hi; mwf_lo = mw0_lo;
    p.num_n_tiles = 0;
    if (!p.h_hi) {
        const int packed_rows = p.o.d_t * Cfg::MP;
        if ((rc = make_map(&mwf_hi, (const __half*)d->wp_hi, packed_rows, H, d->ldwp, Cfg::TILE))) return rc;
        if ((rc = make_map(&mwf_lo, (const __half*)d->wp_lo, packed_rows, H, d->ldwp, Cfg::TILE))) return rc;
        p.num_n_tiles = (p.o.d_t + Cfg::TF - 1) / Cfg::TF;
    }
    const int grid = p.num_m_tiles < sm_count() ? p.num_m_tiles : sm_count();
    NFK_REQUIRE(d->workspace_bytes >= (size_t)grid * (size_t)H * BM * 4, "workspace too small: %zu bytes given, %zu needed",
                d->workspace_bytes, (size_t)grid * (size_t)H * BM * 4);
    bool act = false;                                          // a layer with an activation field: the ACT instance
    for (int l = 0; l < p.num_layers; ++l) act = act || ((p.layer_flags[l] >> SL_ACT_SHIFT) & SL_ACT_MASK) != 0;
    const CUtensorMap maps[8] = {ma_hi, ma_lo, mw0_hi, mw0_lo, mwt_hi, mwt_lo, mwf_hi, mwf_lo};
    return act ? start_step<NB, TAILS, TERMS, true>(maps, grid, p, st) : start_step<NB, TAILS, TERMS, false>(maps, grid, p, st);
}

}  // namespace tc
}  // namespace nfk

using namespace nfk;

extern "C" int nfk_rq_coupling_step_supported(int32_t num_bins, int32_t linear_tails, int32_t hidden_features, int32_t in_features,
                                              int32_t num_square_layers) {
    const bool bins_ok = (num_bins == 8 || num_bins == 10 || num_bins == 4 || num_bins == 16);
    return (bins_ok && hidden_features >= 32 && hidden_features <= tc::STEP_MAX_HIDDEN && hidden_features % 32 == 0 && in_features >= 8 &&
            in_features % 8 == 0 && num_square_layers >= 0 && num_square_layers < tc::STEP_MAX_LAYERS) ? 1 : 0;
}

extern "C" size_t nfk_rq_coupling_step_workspace_bytes(int32_t hidden_features) {
    return (size_t)tc::sm_count() * (size_t)hidden_features * tc::BM * 4;
}

// Checks of the per-row terms, shared by both entry points; *has_terms: `terms` names at least one.
static int check_row_terms(const NfkCouplingStep* d, const NfkStepRowTerms* terms, bool* has_terms) {
    *has_terms = false;
    if (!terms) return NFK_OK;
    for (int l = 0; l < tc::STEP_MAX_LAYERS; ++l) {
        const NfkRowTerm& t = terms->layer[l];
        if (!t.add) continue;
        NFK_REQUIRE(l <= d->num_square_layers, "row term on layer %d, but the trunk has %d layers", l, 1 + d->num_square_layers);
        NFK_REQUIRE(t.ld >= d->hidden_features, "row term of layer %d: ld=%lld is less than the hidden width %d", l, (long long)t.ld,
                    d->hidden_features);
        NFK_REQUIRE(t.ld % 2 == 0 && (reinterpret_cast<uintptr_t>(t.add) & 7) == 0,
                    "row term of layer %d must be 8-byte aligned with an even ld (it is read as float2)", l);
        *has_terms = true;
    }
    NFK_REQUIRE(!*has_terms || d->h_hi == nullptr, "row terms are not supported with the trunk-only output (h_hi)");
    return NFK_OK;
}

// Checks of the trunk's operands, shared by both entry points (its shape has been checked).
static int check_trunk(const NfkCouplingStep* d) {
    NFK_REQUIRE(d->a_hi && d->a_lo && d->w0_hi && d->w0_lo && d->bias_trunk && d->layer_flags && d->workspace, "NULL pointer");
    NFK_REQUIRE(d->num_square_layers == 0 || (d->wt_hi && d->wt_lo && d->wt_exps), "square-layer weights missing");
    NFK_REQUIRE(d->lda % 8 == 0 && d->ldw0 % 8 == 0 && (d->num_square_layers == 0 || d->ldwt % 8 == 0), "row pitches must be multiples of 8");
    NFK_REQUIRE(aligned16(d->a_hi) && aligned16(d->a_lo) && aligned16(d->w0_hi) && aligned16(d->w0_lo) && aligned16(d->bias_trunk) &&
                    aligned16(d->workspace) && (d->num_square_layers == 0 || (aligned16(d->wt_hi) && aligned16(d->wt_lo))),
                "operands must be 16-byte aligned");
    NFK_REQUIRE(d->n_rows < (1ll << 31), "n_rows too large for one launch");
    for (int l = 0; l <= d->num_square_layers; ++l) {
        const int lf = d->layer_flags[l];
        const int e = l == 0 ? d->a_exp + d->w0_exp : d->act_exp + d->wt_exps[l - 1];
        NFK_REQUIRE(!((lf & tc::SL_ADD_SKIP) && (lf & tc::SL_RELU_OUT)), "layer %d: skip add after a relu output is not supported", l);
        NFK_REQUIRE(act_valid(tc::layer_act(lf)), "layer %d: unknown activation code %d in the layer flags", l,
                    (lf >> tc::SL_ACT_SHIFT) & tc::SL_ACT_MASK);
        NFK_REQUIRE(e >= -60 && e <= 60, "scale exponent out of range");
    }
    return NFK_OK;
}

// The trunk's kernel parameters (and the row terms when has_terms).
static void trunk_params(const NfkCouplingStep* d, const NfkStepRowTerms* terms, bool has_terms, tc::StepTermParams& p) {
    const int L = d->num_square_layers;
    memset(&p, 0, sizeof(p));
    p.bias_trunk = d->bias_trunk; p.skip_buf = (float*)d->workspace; p.H = d->hidden_features; p.K0 = d->in_features;
    p.num_layers = 1 + L; p.act_scale = ldexpf(1.0f, d->act_exp);
    for (int l = 0; l <= L; ++l) {
        const int e = l == 0 ? d->a_exp + d->w0_exp : d->act_exp + d->wt_exps[l - 1];
        p.layer_flags[l] = d->layer_flags[l];
        p.acc_scale[l] = ldexpf(1.0f, e);
        p.inv_acc_scale[l] = ldexpf(1.0f, -e);
    }
    p.flags = d->flags; p.n_rows = d->n_rows;
    p.num_m_tiles = (int)((d->n_rows + tc::BM - 1) / tc::BM);
    if (has_terms)
        for (int l = 0; l <= L; ++l) {
            p.add[l] = terms->layer[l].add;
            p.ld_add[l] = terms->layer[l].ld;
        }
}

// The final layer's operands and outputs into the kernel parameters.
static void final_params(const NfkCouplingStep* d, tc::StepTermParams& p) {
    p.o.bias = d->bias_packed; p.o.x = d->x; p.o.y = d->y; p.o.y_hi = (__half*)d->y_hi; p.o.y_lo = (__half*)d->y_lo;
    p.o.t_cols = d->t_cols; p.o.t_col0 = d->t_col0; p.o.out_scale = ldexpf(1.0f, d->y_exp); p.o.ldx = d->ldx; p.o.ldy = d->ldy;
    p.o.lds = d->lds; p.o.d_t = d->d_t; p.o.inverse = d->inverse; p.o.inv_acc_scale = ldexpf(1.0f, -(d->act_exp + d->wp_exp));
    p.lad_accum = d->lad_accum;
}

// The coupling-step launch, with per-row terms on some trunk layers when `terms` is non-null and names at least one.
static int coupling_step(const NfkCouplingStep* d, const NfkStepRowTerms* terms, void* stream) {
    NFK_REQUIRE(d, "NULL descriptor");
    NFK_REQUIRE(d->n_rows >= 0 && d->hidden_features >= 1 && d->in_features >= 1, "bad sizes");
    bool has_terms = false;
    int rc = check_row_terms(d, terms, &has_terms);
    if (rc) return rc;
    if (d->n_rows == 0) return NFK_OK;
    const bool trunk_only = d->h_hi != nullptr;
    const int nb = trunk_only && !d->spline ? 8 : (d->spline ? d->spline->num_bins : 0);
    const int lt = trunk_only && !d->spline ? 1 : (d->spline ? d->spline->linear_tails : 0);
    NFK_REQUIRE(trunk_only || d->spline, "spline descriptor missing");
    NFK_REQUIRE(nfk_rq_coupling_step_supported(nb, lt, d->hidden_features, d->in_features, d->num_square_layers),
                "coupling-step kernel does not take num_bins=%d hidden=%d in_features=%d square layers=%d", nb, d->hidden_features,
                d->in_features, d->num_square_layers);
    if ((rc = check_trunk(d))) return rc;
    if (trunk_only) {
        NFK_REQUIRE(d->h_lo && d->ldh % 8 == 0 && aligned16(d->h_hi) && aligned16(d->h_lo), "bad trunk output pair");
    } else {
        NFK_REQUIRE(d->wp_hi && d->wp_lo && d->bias_packed && d->x && d->d_t >= 1, "NULL pointer");
        NFK_REQUIRE((d->y != nullptr) != (d->y_hi != nullptr), "give either y (fp32 outputs) or y_hi / y_lo (their fp16 split pair)");
        NFK_REQUIRE((d->y_hi == nullptr) == (d->y_lo == nullptr) && d->y_exp >= -60 && d->y_exp <= 60, "bad pair output");
        NFK_REQUIRE(d->t_cols || d->t_col0 >= 0, "t_cols is NULL and t_col0 is negative");
        NFK_REQUIRE(aligned16(d->bias_packed) && aligned16(d->wp_hi) && aligned16(d->wp_lo) && d->ldwp % 8 == 0,
                    "packed final layer must be 16-byte aligned");
        NFK_REQUIRE(d->act_exp + d->wp_exp >= -60 && d->act_exp + d->wp_exp <= 60, "scale exponent out of range");
    }
    tc::StepTermParams p;
    trunk_params(d, terms, has_terms, p);
    cudaStream_t st = (cudaStream_t)stream;
    if (trunk_only) {
        p.h_hi = (__half*)d->h_hi; p.h_lo = (__half*)d->h_lo; p.ldh = d->ldh;
        return tc::launch_step<8, true, false>(d, p, st);
    }
    rc = make_spline_params(d->spline, &p.o.sp);
    if (rc) return rc;
    final_params(d, p);
    const bool tails = d->spline->linear_tails != 0;
#define NFK_STEP(NB)                                                                                      \
    if (has_terms) return tails ? tc::launch_step<NB, true, true>(d, p, st) : tc::launch_step<NB, false, true>(d, p, st); \
    return tails ? tc::launch_step<NB, true, false>(d, p, st) : tc::launch_step<NB, false, false>(d, p, st)
    switch (d->spline->num_bins) {
        case 4: NFK_STEP(4);
        case 8: NFK_STEP(8);
        case 10: NFK_STEP(10);
        case 16: NFK_STEP(16);
    }
#undef NFK_STEP
    return fail(NFK_E_UNSUPPORTED, "num_bins=%d has no coupling-step kernel instance", d->spline->num_bins);
}

extern "C" int nfk_rq_coupling_step_f16x3(const NfkCouplingStep* d, void* stream) { return coupling_step(d, nullptr, stream); }

extern "C" int nfk_rq_coupling_step_terms_f16x3(const NfkCouplingStep* d, const NfkStepRowTerms* terms, void* stream) {
    return coupling_step(d, terms, stream);
}

// The affine epilogue (fused_spline.cuh: AFFINE_NB): the same trunk, terms and workspace; the final layer is MADE's own, 2 d_t
// rows [u_j, shift_j] with no padding, and step->spline is ignored.
extern "C" int nfk_affine_ar_step_f16x3(const NfkCouplingStep* d, const NfkStepRowTerms* terms, void* stream) {
    NFK_REQUIRE(d, "NULL descriptor");
    NFK_REQUIRE(d->n_rows >= 0 && d->hidden_features >= 1 && d->in_features >= 1, "bad sizes");
    NFK_REQUIRE(d->h_hi == nullptr && d->h_lo == nullptr, "the affine step has no trunk-only output (h_hi): use nfk_rq_coupling_step_f16x3");
    bool has_terms = false;
    int rc = check_row_terms(d, terms, &has_terms);
    if (rc) return rc;
    NFK_REQUIRE(d->d_t >= 1 && d->d_t <= (1 << 30), "d_t=%d: the final layer has 2 d_t rows", d->d_t);
    NFK_REQUIRE(d->t_cols == nullptr && d->t_col0 >= 0, "the affine step takes consecutive columns t_col0 .. t_col0 + d_t - 1 (t_cols NULL)");
    NFK_REQUIRE((int64_t)d->t_col0 + d->d_t <= d->ldx && (int64_t)d->t_col0 + d->d_t <= d->ldy,
                "columns t_col0=%d .. + d_t=%d exceed the row pitch of x (%lld) or y (%lld)", d->t_col0, d->d_t, (long long)d->ldx,
                (long long)d->ldy);
    NFK_REQUIRE(d->y != nullptr && d->y_hi == nullptr && d->y_lo == nullptr, "the affine step writes fp32 outputs only (y; no y_hi / y_lo)");
    if (d->n_rows == 0) return NFK_OK;
    NFK_REQUIRE(nfk_rq_coupling_step_supported(8, 1, d->hidden_features, d->in_features, d->num_square_layers),
                "coupling-step kernel does not take hidden=%d in_features=%d square layers=%d", d->hidden_features, d->in_features,
                d->num_square_layers);
    if ((rc = check_trunk(d))) return rc;
    NFK_REQUIRE(d->wp_hi && d->wp_lo && d->bias_packed && d->x, "NULL pointer");
    NFK_REQUIRE(aligned16(d->wp_hi) && aligned16(d->wp_lo) && d->ldwp % 8 == 0, "final-layer weight must be 16-byte aligned");
    NFK_REQUIRE((reinterpret_cast<uintptr_t>(d->bias_packed) & 7) == 0, "final-layer bias must be 8-byte aligned");
    NFK_REQUIRE(d->act_exp + d->wp_exp >= -60 && d->act_exp + d->wp_exp <= 60, "scale exponent out of range");
    tc::StepTermParams p;
    trunk_params(d, terms, has_terms, p);
    final_params(d, p);
    cudaStream_t st = (cudaStream_t)stream;
    return has_terms ? tc::launch_step<tc::AFFINE_NB, false, true>(d, p, st) : tc::launch_step<tc::AFFINE_NB, false, false>(d, p, st);
}

// Rows per feature of the mixture epilogue's packed final layer: roundup(3C, 8), except 48 for C = 11 .. 13, whose 40 rows
// would make an 80-row column tile (the step kernel's MMAs are 96, 112 or 128 wide).  0: C is not supported.
extern "C" int32_t nfk_mog_made_padded_rows(int32_t num_components) {
    if (num_components < 1 || num_components > NFK_MOG_MAX_COMPONENTS) return 0;
    const int mp = (3 * num_components + 7) / 8 * 8;
    return mp == 40 ? 48 : mp;
}

// The mixture epilogue (fused_spline.cuh: mog_tile): the same trunk, terms and workspace; the final layer is MADE's 3C rows per
// feature packed to nfk_mog_made_padded_rows(C), and step->spline is ignored.  One instance per packed row count, always with
// the row terms (none named: p.add[l] is null).
extern "C" int nfk_mog_made_step_f16x3(const NfkCouplingStep* d, const NfkStepRowTerms* terms, const NfkMogArgs* mog, void* stream) {
    NFK_REQUIRE(d && mog, "NULL descriptor");
    NFK_REQUIRE(d->n_rows >= 0 && d->hidden_features >= 1 && d->in_features >= 1, "bad sizes");
    NFK_REQUIRE(d->h_hi == nullptr && d->h_lo == nullptr, "the mixture step has no trunk-only output (h_hi): use nfk_rq_coupling_step_f16x3");
    bool has_terms = false;
    int rc = check_row_terms(d, terms, &has_terms);
    if (rc) return rc;
    const int mp = nfk_mog_made_padded_rows(mog->num_components);
    NFK_REQUIRE(mp > 0, "num_components=%d: the mixture step takes 1 .. %d components", mog->num_components, NFK_MOG_MAX_COMPONENTS);
    NFK_REQUIRE(mog->epsilon > 0.0f && mog->epsilon < INFINITY, "epsilon=%g must be positive and finite", (double)mog->epsilon);
    NFK_REQUIRE(mog->mode == NFK_MOG_LOG_PROB || mog->mode == NFK_MOG_SAMPLE, "mode=%d is neither NFK_MOG_LOG_PROB nor NFK_MOG_SAMPLE",
                mog->mode);
    const bool sample = mog->mode == NFK_MOG_SAMPLE;
    NFK_REQUIRE(d->d_t >= 1 && d->d_t <= (1 << 30), "d_t=%d: the final layer has d_t features", d->d_t);
    NFK_REQUIRE(d->t_cols == nullptr && d->t_col0 >= 0, "the mixture step takes consecutive columns t_col0 .. t_col0 + d_t - 1 (t_cols NULL)");
    NFK_REQUIRE(d->y_hi == nullptr && d->y_lo == nullptr, "the mixture step writes fp32 outputs only (no y_hi / y_lo)");
    if (sample) {
        NFK_REQUIRE(d->y && mog->u && mog->e, "sample mode needs y and the noise u, e");
        NFK_REQUIRE(d->lad_accum == nullptr, "sample mode writes y only (lad_accum must be NULL)");
        NFK_REQUIRE((int64_t)d->t_col0 + d->d_t <= d->ldy && mog->ld_noise >= d->d_t,
                    "columns t_col0=%d .. + d_t=%d exceed the row pitch of y (%lld), or ld_noise=%lld < d_t", d->t_col0, d->d_t,
                    (long long)d->ldy, (long long)mog->ld_noise);
    } else {
        NFK_REQUIRE(d->x && d->lad_accum, "log_prob mode needs x and lad_accum");
        NFK_REQUIRE(d->y == nullptr && mog->u == nullptr && mog->e == nullptr, "log_prob mode takes no y and no noise (u, e NULL)");
        NFK_REQUIRE((int64_t)d->t_col0 + d->d_t <= d->ldx, "columns t_col0=%d .. + d_t=%d exceed the row pitch of x (%lld)", d->t_col0,
                    d->d_t, (long long)d->ldx);
    }
    if (d->n_rows == 0) return NFK_OK;
    NFK_REQUIRE(nfk_rq_coupling_step_supported(8, 1, d->hidden_features, d->in_features, d->num_square_layers),
                "coupling-step kernel does not take hidden=%d in_features=%d square layers=%d", d->hidden_features, d->in_features,
                d->num_square_layers);
    if ((rc = check_trunk(d))) return rc;
    NFK_REQUIRE(d->wp_hi && d->wp_lo && d->bias_packed, "NULL pointer");
    NFK_REQUIRE(aligned16(d->bias_packed) && aligned16(d->wp_hi) && aligned16(d->wp_lo) && d->ldwp % 8 == 0,
                "packed final layer must be 16-byte aligned");
    NFK_REQUIRE(d->act_exp + d->wp_exp >= -60 && d->act_exp + d->wp_exp <= 60, "scale exponent out of range");
    tc::StepMogParams p;
    trunk_params(d, terms, has_terms, p);
    final_params(d, p);
    if (sample) p.o.x = nullptr;                     // not read
    p.mog.u = mog->u; p.mog.e = mog->e; p.mog.ldn = mog->ld_noise; p.mog.eps = mog->epsilon; p.mog.C = mog->num_components;
    p.mog.sample = sample;
    cudaStream_t st = (cudaStream_t)stream;
    switch (mp) {
        case 8: return tc::launch_step<tc::mog_nb(8), false, true>(d, p, st);
        case 16: return tc::launch_step<tc::mog_nb(16), false, true>(d, p, st);
        case 24: return tc::launch_step<tc::mog_nb(24), false, true>(d, p, st);
        case 32: return tc::launch_step<tc::mog_nb(32), false, true>(d, p, st);
        case 48: return tc::launch_step<tc::mog_nb(48), false, true>(d, p, st);
        case 56: return tc::launch_step<tc::mog_nb(56), false, true>(d, p, st);
        case 64: return tc::launch_step<tc::mog_nb(64), false, true>(d, p, st);
    }
    return fail(NFK_E_UNSUPPORTED, "num_components=%d has no mixture-step instance", mog->num_components);
}

#ifdef NFK_STEP_CLOCKS
// Phase-clock builds only (scripts/step_phases.py): the stamp buffer's shape {CTAs, rounds, column tiles, stamps per tile}
// into dims and, when dst is not null, the buffer of the last stamped launch into host memory: per (CTA, round) 4 trunk stamps
// (warpgroup 0 start / end, warpgroup 1 start / end), then the stamps of each column tile.  0 on success.
extern "C" int nfk_step_clocks(long long* dst, int32_t* dims) {
    dims[0] = tc::CLK_CTAS; dims[1] = tc::CLK_ROUNDS; dims[2] = tc::CLK_TILES; dims[3] = tc::CLK_TILE_STAMPS;
    if (!dst) return 0;
    return cudaMemcpyFromSymbol(dst, tc::g_step_clocks, sizeof(tc::g_step_clocks)) == cudaSuccess ? 0 : -1;
}
#endif
