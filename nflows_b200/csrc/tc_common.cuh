// wgmma / TMA / mbarrier building blocks shared by the tensor-core kernels of libnfk_sm90.so (inline PTX for sm_90a).
//
// Every tensor-core kernel of the library has the same shape: one persistent CTA per SM, 384 threads.
//   warpgroup 0      : TMA producer -- one elected thread streams [A hi | A lo | W hi | W lo] K-slabs (2-D boxes of fp16,
//                      SWIZZLE_64B, out-of-bounds rows / columns zero-filled by the TMA unit) into a ring of STAGES slots
//   warpgroups 1 - 2 : consumers -- each multiplies ITS 64 rows of the 128-row A tile with the 128-row W tile
//                      (wgmma m64n128k16, both operands K-major from shared memory) and runs the epilogue on the
//                      accumulators it holds in registers (the coupling-step kernel's final layer departs from this: one
//                      warpgroup per column tile, nfk_coupling_step_tc.cu)
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "nfk_common.cuh"

namespace nfk {
namespace tc {

constexpr int BM = 128;            // rows per tile: two consumer warpgroups x 64 rows
constexpr int BN = 128;            // columns per tile = wgmma N
constexpr int BK = 32;             // fp16 elements per K-slab = one 64-byte swizzle row (SWIZZLE_64B) = two wgmma K-steps
constexpr int THREADS = 384;       // warpgroup 0: TMA producer; warpgroups 1-2: wgmma + epilogue
constexpr int A_BYTES = BM * BK * 2;                      // 8 KB
constexpr int B_BYTES = BN * BK * 2;                      // 8 KB
constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;    // 32 KB: [A hi | A lo | W hi | W lo]
constexpr int ROW_BYTES = BK * 2;
// K-slabs accumulated by the tensor core before the partial sum is added to the running sums (precision vs. register moves):
constexpr int DRAIN_SLABS_LINEAR = 2;   // dense layers: K = 64 (12 MMAs) -- their outputs feed log p directly
constexpr int DRAIN_SLABS_FUSED = 4;    // fused coupling: K = 128 (24 MMAs) -- its outputs are spline logits

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// One lane of a converged warp (elect.sync): keeps the producer role on the uniform datapath.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "elect.sync _|P1, 0xffffffff;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}\n"
        : "+r"(pred));
    return pred != 0;
}
// named barrier of one consumer warpgroup (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }
// named barrier `id` shared by both consumer warpgroups (256 threads): one side signals, the other waits
__device__ __forceinline__ void pair_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void pair_wait(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// d[N / 2] (+)= A[64 x 16] * B[N x 16]^T, fp16 inputs, fp32 accumulators; accumulate == 0 overwrites d.  N = 128 everywhere
// but the final layer of the coupling-step kernel, whose column tiles are FusedCfg::TILE (96 or 112) packed rows wide.
// Fragment layout of d (per thread of the warpgroup, warp wi, lane l): d[i] is row 16 wi + l/4 + 8 ((i >> 1) & 1),
// column 8 (i >> 2) + 2 (l & 3) + (i & 1).
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<112>(float (&d)[56], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %58, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n112k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55}, "
        "%56, %57, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<96>(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %50, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
        "%48, %49, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

// K-major SWIZZLE_64B shared-memory matrix descriptor (sm_90 wgmma): [0,14) start >> 4 | [16,30) LBO >> 4 (unused for
// swizzled K-major, 1) | [32,46) SBO >> 4 = 8 rows x 64 bytes | [62,64) layout 2 = SWIZZLE_64B.  A K-step of 16 fp16 = 32 bytes
// advances the start address by 2.
static_assert(ROW_BYTES == 64, "descriptors assume 64-byte K-slab rows");
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)((8 * ROW_BYTES) >> 4) << 32) | (2ull << 62);
}

// Ring of STAGE_BYTES slots filled by the producer; `full` barriers complete on the TMA bytes, `empty` barriers collect one
// arrival per consumer warp (8).
struct Ring {
    uint32_t base, full, empty;
    int stages;
    uint32_t stage_bytes;
    int stage = 0;
    uint32_t phase = 0;
    __device__ __forceinline__ void advance() {
        if (++stage == stages) { stage = 0; phase ^= 1; }
    }
};

// Producer: one K-slab of the A rows [m0, m0 + 128) and the W rows [n0, n0 + 128) into the next ring slot.
__device__ __forceinline__ void produce_slab(Ring& r, const CUtensorMap* a_hi, const CUtensorMap* a_lo, const CUtensorMap* w_hi,
                                             const CUtensorMap* w_lo, int ks, int m0, int n0) {
    mbar_wait(r.empty + 8 * r.stage, r.phase ^ 1);
    const uint32_t full = r.full + 8 * r.stage;
    const uint32_t sa = r.base + r.stage * r.stage_bytes;
    mbar_expect_tx(full, STAGE_BYTES);
    tma_load_2d(sa, a_hi, full, ks * BK, m0);
    tma_load_2d(sa + A_BYTES, a_lo, full, ks * BK, m0);
    tma_load_2d(sa + 2 * A_BYTES, w_hi, full, ks * BK, n0);
    tma_load_2d(sa + 2 * A_BYTES + B_BYTES, w_lo, full, ks * BK, n0);
    r.advance();
}

// Producer, weights only: one K-slab of the W rows [n0, n0 + rows) into the next slot of a ring of [W hi | W lo] slots (W lo
// at lo_off; rows is the box height of both maps, <= BN).
__device__ __forceinline__ void produce_w_slab(Ring& r, const CUtensorMap* w_hi, const CUtensorMap* w_lo, int ks, int n0, int rows = BN,
                                               uint32_t lo_off = B_BYTES) {
    mbar_wait(r.empty + 8 * r.stage, r.phase ^ 1);
    const uint32_t full = r.full + 8 * r.stage;
    const uint32_t sw = r.base + r.stage * r.stage_bytes;
    mbar_expect_tx(full, 2 * rows * ROW_BYTES);
    tma_load_2d(sw, w_hi, full, ks * BK, n0);
    tma_load_2d(sw + lo_off, w_lo, full, ks * BK, n0);
    r.advance();
}

// Consumer warpgroup `wg`: the tile's num_k K-slabs added to the running sums.  Per K-step the two small cross terms
// (a_lo w_hi, a_hi w_lo), then the main product a_hi w_hi, into one fp32 accumulator (the dropped a_lo w_lo term is ~2^-22
// relative).  The tensor core adds with round-toward-zero, so a partial sum covers only `drain` slabs before it is added to
// `sum` with round-to-nearest.  One slab's MMAs stay in flight while the next slab's are issued.
// Streamed A (a_res == 0): ring slots hold [A hi | A lo | W hi | W lo].  Resident A: K-slab ks of A is the [hi | lo] pair at
// a_res + ks * 2 * A_BYTES (same 128-row SWIZZLE_64B layout) and the ring slots hold [W hi | W lo].
__device__ __forceinline__ void mma_tile(float (&sum)[64], Ring& r, int num_k, int drain, int wg, int lane, uint32_t a_res = 0) {
    float acc[64];
    for (int g0 = 0; g0 < num_k; g0 += drain) {
        const int slabs = min(drain, num_k - g0);
        int prev = -1;
        for (int j = 0; j < slabs; ++j) {
            mbar_wait(r.full + 8 * r.stage, r.phase);
            const uint32_t ss = r.base + r.stage * r.stage_bytes;
            const uint32_t sa = a_res ? a_res + (uint32_t)(g0 + j) * 2 * A_BYTES : ss;
            const uint32_t sw = a_res ? ss : ss + 2 * A_BYTES;
            const uint64_t a_hi = make_smem_desc(sa + wg * (A_BYTES / 2)), a_lo = make_smem_desc(sa + A_BYTES + wg * (A_BYTES / 2));
            const uint64_t w_hi = make_smem_desc(sw), w_lo = make_smem_desc(sw + B_BYTES);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < BK / 16; ++kk) {
                const uint64_t adv = (uint64_t)(kk * 2);
                wgmma_f16<BN>(acc, a_lo + adv, w_hi + adv, (j | kk) != 0);
                wgmma_f16<BN>(acc, a_hi + adv, w_lo + adv, 1);
            }
#pragma unroll
            for (int kk = 0; kk < BK / 16; ++kk) {
                const uint64_t adv = (uint64_t)(kk * 2);
                wgmma_f16<BN>(acc, a_hi + adv, w_hi + adv, 1);
            }
            wgmma_commit();
            if (prev >= 0) {
                wgmma_wait<1>();
                __syncwarp();
                if (lane == 0) mbar_arrive(r.empty + 8 * prev);
            }
            prev = r.stage;
            r.advance();
        }
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(r.empty + 8 * prev);
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = __fadd_rn(sum[i], acc[i]);
    }
}

// Split of one fp32 value into the fp16 pair the kernels multiply with: v * scale = hi + lo (+ <= 2^-22 relative), hi the
// nearest fp16, lo the nearest fp16 of the exact remainder.  |v * scale| beyond the fp16 range raises NFK_FLAG_F16_RANGE.
__device__ __forceinline__ void split_f16(float v, float scale, __half& hi, __half& lo, int& flag) {
    const float s = v * scale;
    if (!(fabsf(s) <= 65000.0f)) flag |= 4;
    hi = __float2half_rn(s);
    lo = __float2half_rn(s - __half2float(hi));
}

// host helpers (nfk_linear_tc.cu)
int make_map(CUtensorMap* map, const __half* base, int64_t rows, int K, int64_t ld, int box_rows);

}  // namespace tc
}  // namespace nfk
