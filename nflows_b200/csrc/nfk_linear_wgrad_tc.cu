// Backward of the split-fp16 dense layer (training of a conditioner on the tensor cores): the weight / bias gradient
//
//   dW[o, i] = sum_b G[b, o] A[b, i]        db[o] = sum_b G[b, o]
//
// on wgmma with the arithmetic of nfk_linear_f16x3 (three MMAs per K-step on split pairs, partial sums drained to registers
// with round-to-nearest adds), and the pass that turns the gradient of a layer's input into the split pair of the gradient of
// the layer in front of it (relu mask, skip connection, split).
//
// Both operands of the weight gradient are row-major [batch, features] pairs, so for this product (M = out, N = in, K = batch)
// both are MN-major.  The producer warpgroup transposes while it stages: it reads 32 batch rows x 128 feature columns of each
// matrix with coalesced half2 loads and writes them to the ring slot as the K-major SWIZZLE_64B tile a TMA load of a [128, 32]
// box would have written, so the consumers run tc_common.cuh's mma_tile unchanged.  The bias gradient is one more column of the
// B operand would cost a whole extra tile at in = 128, so it is a plain column sum of the gradient pair instead (bias_partial_kernel),
// over the same slabs.
//
// Determinism: the batch is cut into slabs whose size depends on (n_rows, out, in) only (wgrad_slab_rows); each (slab, 128 x 128
// tile) work item writes its partial sums to its own workspace block (tile-padded, so the epilogue stores without bounds checks),
// and a second pass adds the slabs in slab order.  Every
// partial is a fixed sequence of MMAs and adds, so the result is bitwise identical across repeats, launch geometries and devices.
#include <stdlib.h>

#include "tc_common.cuh"

namespace nfk {
namespace tc {

constexpr int WG_STAGES = 6;                                              // 6 x 32 KB ring, as the dense layer
constexpr int WG_SMEM_BYTES = WG_STAGES * STAGE_BYTES + 256 /*barriers*/ + 1024 /*alignment slack*/;
constexpr int WG_PRODUCERS = 128;                                          // warpgroup 0 stages every slot
constexpr int WG_MIN_SLAB = 512;                                           // batch rows per slab, at least
constexpr int WG_TARGET_ITEMS = 512;                                       // (slab, tile) work items aimed at per launch

struct WgradParams {
    const __half* g_hi; const __half* g_lo; int64_t ldg;     // [n_rows, out]
    const __half* a_hi; const __half* a_lo; int64_t lda;     // [n_rows, in]
    float* ws;                                                 // [num_slabs][num_m_tiles * BM][num_n_tiles * BN]
    float inv_scale;                                           // 2^-(g_exp + a_exp)
    int64_t n_rows;
    int slab_rows, num_slabs;
    int out, in;
    int num_m_tiles, num_n_tiles;
    int vec_g, vec_a;                                          // half2 loads allowed (even pitch, 4-byte aligned bases)
};

// One operand tile of a ring slot: rows = feature columns [c0, c0 + 128) of a row-major [n_rows, ncols] fp16 matrix, K = its batch
// rows [kb, kb + 32) (zero at and beyond kend), written K-major with the 64-byte swizzle of the TMA maps (16-byte chunk q of row r
// at chunk q ^ ((r >> 1) & 3)).  Thread t of the producer warpgroup stages rows 2 (t & 63), + 1 and K-chunks 2 (t >> 6), + 1.
__device__ __forceinline__ void stage_transposed(uint32_t dst, const __half* __restrict__ src, int64_t ld, int ncols, int c0,
                                                 int64_t kb, int64_t kend, bool vec) {
    const int t = threadIdx.x;
    const int cp = t & 63, bh = t >> 6;
    const int c = c0 + 2 * cp;
    const __half* row0 = src + (kb + 16 * bh) * ld + c;
    uint32_t v[16];
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
        const int64_t b = kb + 16 * bh + kk;
        uint32_t x = 0u;                                     // the half2 (column c, column c + 1) as bits
        if (b < kend) {
            const __half* p = row0 + kk * ld;
            if (vec && c + 1 < ncols) {
                x = __ldg(reinterpret_cast<const unsigned int*>(p));
            } else {
                uint32_t e0 = 0u, e1 = 0u;
                if (c < ncols) e0 = __half_as_ushort(p[0]);
                if (c + 1 < ncols) e1 = __half_as_ushort(p[1]);
                x = e0 | (e1 << 16);
            }
        }
        v[kk] = x;
    }
    const int sw = cp & 3;                                   // (row >> 1) & 3 of both rows
#pragma unroll
    for (int h = 0; h < 2; ++h) {                            // row 2 cp + h takes half h of every pair
        const uint32_t sel = h ? 0x7632u : 0x5410u;
        const uint32_t row = dst + (uint32_t)(2 * cp + h) * ROW_BYTES;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int kq = 8 * q;
            const uint32_t w0 = __byte_perm(v[kq + 0], v[kq + 1], sel), w1 = __byte_perm(v[kq + 2], v[kq + 3], sel);
            const uint32_t w2 = __byte_perm(v[kq + 4], v[kq + 5], sel), w3 = __byte_perm(v[kq + 6], v[kq + 7], sel);
            const uint32_t addr = row + (uint32_t)(((2 * bh + q) ^ sw) * 16);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(w0), "r"(w1), "r"(w2), "r"(w3) : "memory");
        }
    }
}

__global__ void __launch_bounds__(THREADS, 1) linear_wgrad_kernel(const WgradParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bars = smem_base + WG_STAGES * STAGE_BYTES;
    Ring ring{smem_base, bars, bars + 8 * WG_STAGES, WG_STAGES, (uint32_t)STAGE_BYTES};
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles = p.num_m_tiles * p.num_n_tiles;
    const int items = tiles * p.num_slabs;

    if (threadIdx.x == 0) {
        for (int s = 0; s < WG_STAGES; ++s) { mbar_init(ring.full + 8 * s, WG_PRODUCERS); mbar_init(ring.empty + 8 * s, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 72;" ::: "memory");
        // ================================================= producers: transpose-and-stage every K-slab of every work item
        for (int t = blockIdx.x; t < items; t += gridDim.x) {
            const int slab = t / tiles, tile = t % tiles;
            const int m0 = (tile / p.num_n_tiles) * BM, n0 = (tile % p.num_n_tiles) * BN;
            const int64_t b0 = (int64_t)slab * p.slab_rows;
            const int64_t b1 = min(p.n_rows, b0 + p.slab_rows);
            const int num_k = (int)((b1 - b0 + BK - 1) / BK);
            for (int ks = 0; ks < num_k; ++ks) {
                mbar_wait(ring.empty + 8 * ring.stage, ring.phase ^ 1);
                const uint32_t sa = ring.base + ring.stage * ring.stage_bytes;
                const int64_t kb = b0 + (int64_t)ks * BK;
                // [G hi | G lo | A hi | A lo], one tile at a time (16 loads in flight per thread: the producers' register budget)
#pragma unroll 1
                for (int m = 0; m < 4; ++m) {
                    const bool is_g = m < 2;
                    const __half* src = m == 0 ? p.g_hi : m == 1 ? p.g_lo : m == 2 ? p.a_hi : p.a_lo;
                    stage_transposed(sa + m * A_BYTES, src, is_g ? p.ldg : p.lda, is_g ? p.out : p.in, is_g ? m0 : n0, kb, b1,
                                     is_g ? p.vec_g : p.vec_a);
                }
                // the tiles were written through the generic proxy; wgmma reads them through the async proxy
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                mbar_arrive(ring.full + 8 * ring.stage);
                ring.advance();
            }
        }
        return;
    }
    // ================================================= consumers: warpgroup wg owns output rows [64 wg, 64 wg + 64) of every tile
    asm volatile("setmaxnreg.inc.sync.aligned.u32 216;" ::: "memory");
    const int wg = (warp >> 2) - 1, wi = warp & 3;
    const int q = lane & 3;
    for (int t = blockIdx.x; t < items; t += gridDim.x) {
        const int slab = t / tiles, tile = t % tiles;
        const int m0 = (tile / p.num_n_tiles) * BM, n0 = (tile % p.num_n_tiles) * BN;
        const int64_t b0 = (int64_t)slab * p.slab_rows;
        const int64_t b1 = min(p.n_rows, b0 + p.slab_rows);
        const int num_k = (int)((b1 - b0 + BK - 1) / BK);
        float sum[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = 0.0f;
        mma_tile(sum, ring, num_k, DRAIN_SLABS_LINEAR, wg, lane);
        const int ldw = p.num_n_tiles * BN;
        float* wr = p.ws + ((int64_t)slab * p.num_m_tiles * BM + m0 + wg * 64 + wi * 16 + (lane >> 2)) * ldw + n0 + 2 * q;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 16; ++j)
                *reinterpret_cast<float2*>(wr + 8 * h * ldw + 8 * j) =
                    make_float2(sum[4 * j + 2 * h] * p.inv_scale, sum[4 * j + 2 * h + 1] * p.inv_scale);
    }
}

// Bias-gradient partials: wsb[slab, o] = the sum over the slab's rows of the gradient pair's value (hi + lo) 2^-g_exp.  A block
// takes 32 columns of one slab: thread (ty, tx) adds rows ty, ty + 8, ... of column tx in row order, then ty = 0 adds the eight
// sums in order -- a fixed order, whatever the launch geometry.
__global__ void __launch_bounds__(256) bias_partial_kernel(const __half* __restrict__ g_hi, const __half* __restrict__ g_lo, int64_t ldg,
                                                           float inv_scale, int64_t n_rows, int slab_rows, int num_slabs, int out,
                                                           float* __restrict__ wsb) {
    __shared__ float part[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int groups = (out + 31) / 32;
    for (int64_t item = blockIdx.x; item < (int64_t)num_slabs * groups; item += gridDim.x) {
        const int slab = (int)(item / groups), o = (int)(item - (int64_t)slab * groups) * 32 + tx;
        const int64_t b0 = (int64_t)slab * slab_rows, b1 = min(n_rows, b0 + slab_rows);
        float s = 0.0f;
        if (o < out)
            for (int64_t b = b0 + ty; b < b1; b += 8)
                s = __fadd_rn(s, __fadd_rn(__half2float(g_hi[b * ldg + o]), __half2float(g_lo[b * ldg + o])) * inv_scale);
        part[ty][tx] = s;
        __syncthreads();
        if (ty == 0 && o < out) {
            float t = 0.0f;
#pragma unroll
            for (int k = 0; k < 8; ++k) t = __fadd_rn(t, part[k][tx]);
            wsb[(int64_t)slab * out + o] = t;
        }
        __syncthreads();
    }
}

// dW / db = the slabs' partial sums added in slab order (0 slabs: zero gradients).  ws: [num_slabs][rows_pad][cols_pad] of the
// weight, wsb: [num_slabs][out] of the bias (db NULL: not read).
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ ws, const float* __restrict__ wsb, int num_slabs,
                                                           int out, int in, int rows_pad, int cols_pad, float* __restrict__ dw,
                                                           int64_t ldw, float* __restrict__ db) {
    const int cols = in + (db ? 1 : 0);
    const int64_t total = (int64_t)out * cols, slab_stride = (int64_t)rows_pad * cols_pad;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int o = (int)(idx / cols), i = (int)(idx - (int64_t)o * cols);
        float s = 0.0f;
        if (i < in) {
            for (int k = 0; k < num_slabs; ++k) s = __fadd_rn(s, __ldcs(ws + k * slab_stride + (int64_t)o * cols_pad + i));
            dw[(int64_t)o * ldw + i] = s;
        } else {
            for (int k = 0; k < num_slabs; ++k) s = __fadd_rn(s, wsb[(int64_t)k * out + o]);
            db[o] = s;
        }
    }
}

// G = dA (x) [mask != 0] + skip as the split pair of exponent `scale` (and fp32 when g is given); columns [n_cols, n_cols_pad)
// of the pair are written as zeros.
__global__ void __launch_bounds__(256) mask_split_kernel(const float* __restrict__ da, int64_t ldd, const __half* __restrict__ m_hi,
                                                         const __half* __restrict__ m_lo, int64_t ldm, const float* __restrict__ skip,
                                                         int64_t ldk, int n_cols, int n_cols_pad, float scale, __half* __restrict__ hi,
                                                         __half* __restrict__ lo, int64_t ldo, float* __restrict__ g, int64_t ldg,
                                                         int64_t n_rows, int32_t* flags) {
    int flag = 0;
    const int64_t total = n_rows * n_cols_pad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / n_cols_pad;
        const int j = (int)(i - r * n_cols_pad);
        __half h = __float2half_rn(0.0f), l = h;
        if (j < n_cols) {
            float v = __ldcs(da + r * ldd + j);
            if (m_hi && ((__half_as_ushort(m_hi[r * ldm + j]) | __half_as_ushort(m_lo[r * ldm + j])) & 0x7fff) == 0) v = 0.0f;
            if (skip) v += skip[r * ldk + j];
            if (g) g[r * ldg + j] = v;
            split_f16(v, scale, h, l, flag);
        }
        hi[r * ldo + j] = h;
        lo[r * ldo + j] = l;
    }
    if (flag && flags) atomicOr(flags, flag);
}

// Batch rows per slab: a multiple of BK, at least WG_MIN_SLAB, enough slabs for about WG_TARGET_ITEMS work items.  A function of
// the shape alone, never of the device.
static int wgrad_slab_rows(int64_t n_rows, int tiles) {
    const int64_t want = (WG_TARGET_ITEMS + tiles - 1) / tiles;
    int64_t s = (n_rows + want - 1) / want;
    s = (s + BK - 1) / BK * BK;
    if (s < WG_MIN_SLAB) s = WG_MIN_SLAB;
    if (s > (1 << 30)) s = 1 << 30;
    return (int)s;
}

static void wgrad_shape(int64_t n_rows, int out, int in, int* m_tiles, int* n_tiles, int* slab, int* slabs) {
    *m_tiles = (out + BM - 1) / BM;
    *n_tiles = (in + BN - 1) / BN;
    *slab = wgrad_slab_rows(n_rows, *m_tiles * *n_tiles);
    *slabs = (int)((n_rows + *slab - 1) / *slab);
}

}  // namespace tc
}  // namespace nfk

using namespace nfk;

static bool wgrad_exp_ok(int e) { return e >= -60 && e <= 60; }

static bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return a && b && na && nb && x < y + nb && y < x + na;
}

extern "C" size_t nfk_linear_f16x3_wgrad_workspace(int64_t n_rows, int32_t out_features, int32_t in_features, int want_bias) {
    if (n_rows <= 0 || out_features < 1 || in_features < 1) return 0;
    int mt, nt, slab, slabs;
    tc::wgrad_shape(n_rows, out_features, in_features, &mt, &nt, &slab, &slabs);
    return (size_t)slabs * ((size_t)mt * tc::BM * (size_t)nt * tc::BN + (want_bias ? (size_t)out_features : 0)) * sizeof(float);
}

extern "C" int nfk_linear_f16x3_wgrad(const void* g_hi, const void* g_lo, int64_t ldg, int32_t g_exp, const void* a_hi,
                                      const void* a_lo, int64_t lda, int32_t a_exp, float* dw, int64_t ldw, float* db,
                                      int64_t n_rows, int32_t out_features, int32_t in_features, void* workspace,
                                      size_t workspace_bytes, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && out_features >= 1 && in_features >= 1, "bad sizes n_rows=%lld out=%d in=%d", (long long)n_rows,
                out_features, in_features);
    NFK_REQUIRE(dw, "NULL dW");
    NFK_REQUIRE(ldw >= in_features, "ldw=%lld < in_features=%d", (long long)ldw, in_features);
    NFK_REQUIRE(wgrad_exp_ok(g_exp) && wgrad_exp_ok(a_exp), "scale exponent out of range");
    int mt, nt, slab, slabs;
    tc::wgrad_shape(n_rows, out_features, in_features, &mt, &nt, &slab, &slabs);
    const size_t need = nfk_linear_f16x3_wgrad_workspace(n_rows, out_features, in_features, db != nullptr);
    NFK_REQUIRE(workspace_bytes >= need && (need == 0 || workspace), "workspace of %zu bytes, need %zu (nfk_linear_f16x3_wgrad_workspace)",
                workspace_bytes, need);
    const size_t dw_bytes = ((size_t)(out_features - 1) * (size_t)ldw + (size_t)in_features) * sizeof(float);
    NFK_REQUIRE(!overlaps(dw, dw_bytes, workspace, need) && !overlaps(db, (size_t)out_features * 4, workspace, need) &&
                    !overlaps(dw, dw_bytes, db, (size_t)out_features * 4),
                "dW, db and the workspace must not overlap");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_rows > 0) {
        NFK_REQUIRE(g_hi && g_lo && a_hi && a_lo, "NULL operand pointer");
        NFK_REQUIRE(ldg >= out_features && lda >= in_features, "row pitches must cover the features (ldg=%lld, lda=%lld)",
                    (long long)ldg, (long long)lda);
        tc::WgradParams p;
        p.g_hi = (const __half*)g_hi; p.g_lo = (const __half*)g_lo; p.ldg = ldg;
        p.a_hi = (const __half*)a_hi; p.a_lo = (const __half*)a_lo; p.lda = lda;
        p.ws = (float*)workspace;
        p.inv_scale = ldexpf(1.0f, -(g_exp + a_exp));
        p.n_rows = n_rows; p.slab_rows = slab; p.num_slabs = slabs;
        p.out = out_features; p.in = in_features;
        p.num_m_tiles = mt; p.num_n_tiles = nt;
        auto al4 = [](const void* q) { return ((uintptr_t)q & 3u) == 0; };
        p.vec_g = (ldg % 2 == 0) && al4(g_hi) && al4(g_lo);
        p.vec_a = (lda % 2 == 0) && al4(a_hi) && al4(a_lo);
        static DeviceOnce attr_once;
        int attr_dev = 0;
        if (attr_once.pending(&attr_dev)) {
            cudaError_t e = cudaFuncSetAttribute(tc::linear_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::WG_SMEM_BYTES);
            if (e != cudaSuccess) return fail(NFK_E_CUDA, "cudaFuncSetAttribute(smem=%d): %s", tc::WG_SMEM_BYTES, cudaGetErrorString(e));
            attr_once.mark(attr_dev);
        }
        const int64_t items = (int64_t)mt * nt * slabs;
        const int grid = (int)(items < tc::sm_count() ? items : tc::sm_count());
        tc::linear_wgrad_kernel<<<grid, tc::THREADS, tc::WG_SMEM_BYTES, st>>>(p);
        if (int rc = check_launch("linear_wgrad_kernel")) return rc;
    }
    const int64_t cap = (int64_t)tc::sm_count() * 8;
    float* wsb = (float*)workspace + (size_t)slabs * mt * tc::BM * nt * tc::BN;
    if (db && n_rows > 0) {
        const int64_t blocks = (int64_t)slabs * ((out_features + 31) / 32);
        tc::bias_partial_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>((const __half*)g_hi, (const __half*)g_lo, ldg,
                                                                                  ldexpf(1.0f, -g_exp), n_rows, slab, slabs,
                                                                                  out_features, wsb);
        if (int rc = check_launch("bias_partial_kernel")) return rc;
    }
    const int64_t blocks = ((int64_t)out_features * (in_features + 1) + 255) / 256;
    tc::wgrad_reduce_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>((const float*)workspace, wsb, slabs, out_features,
                                                                              in_features, mt * tc::BM, nt * tc::BN, dw, ldw, db);
    return check_launch("wgrad_reduce_kernel");
}

extern "C" int nfk_mask_split_f16(const float* da, int64_t ldd, const void* mask_hi, const void* mask_lo, int64_t ldm,
                                  const float* skip, int64_t ldk, int32_t n_cols, int32_t n_cols_pad, int32_t scale_exp,
                                  void* g_hi, void* g_lo, int64_t ldo, float* g, int64_t ldg, int64_t n_rows, int32_t* flags,
                                  void* stream) {
    NFK_REQUIRE(n_rows >= 0 && n_cols >= 1 && n_cols_pad >= n_cols && wgrad_exp_ok(scale_exp), "bad sizes");
    NFK_REQUIRE((mask_hi == nullptr) == (mask_lo == nullptr), "mask_hi and mask_lo must be given together");
    NFK_REQUIRE(ldd >= n_cols && ldo >= n_cols_pad && (!mask_hi || ldm >= n_cols) && (!skip || ldk >= n_cols) &&
                    (!g || ldg >= n_cols),
                "row pitches must cover the columns");
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(da && g_hi && g_lo, "NULL pointer");
    NFK_REQUIRE((const void*)g != (const void*)da, "g must not alias dA");
    const int64_t blocks = (n_rows * n_cols_pad + 255) / 256, cap = (int64_t)tc::sm_count() * 32;
    tc::mask_split_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream>>>(
        da, ldd, (const __half*)mask_hi, (const __half*)mask_lo, ldm, skip, ldk, n_cols, n_cols_pad, ldexpf(1.0f, scale_exp),
        (__half*)g_hi, (__half*)g_lo, ldo, g, ldg, n_rows, flags);
    return check_launch("mask_split_kernel");
}
