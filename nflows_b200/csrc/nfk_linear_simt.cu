// Dense layer Y = post(pre(X) W^T + b) + R (pre, post: activation codes, include/nfk.h) on the FP32 FFMA pipe (exact fp32 products, fp32 accumulate).
// This is the precision-reference GEMM of the path (bit-comparable to an fp32 sgemm up to summation order) and the
// fallback for shapes the wgmma split-fp16 kernel does not take.  128x128x16 tiles, 8x8 register micro-tiles,
// global->register prefetch of the next K-slab while the current one is consumed from shared memory.
#include "nfk_common.cuh"

namespace nfk {

constexpr int BM = 128, BN = 128, BK = 16, PAD = 4, GEMM_THREADS = 256;

__device__ __forceinline__ void load8(const float* __restrict__ base, int64_t ld, int64_t row, int64_t n_rows, int k,
                                      int K, bool vec_ok, int act, float (&v)[8]) {
    if (row < n_rows) {
        const float* p = base + row * ld + k;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (vec_ok && k + 4 * h + 3 < K) {
                float4 t = __ldg(reinterpret_cast<const float4*>(p + 4 * h));
                v[4 * h + 0] = t.x; v[4 * h + 1] = t.y; v[4 * h + 2] = t.z; v[4 * h + 3] = t.w;
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) v[4 * h + i] = (k + 4 * h + i < K) ? __ldg(p + 4 * h + i) : 0.0f;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = 0.0f;
    }
    if (act) {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = nfk_act(act, v[i]);
    }
}

__global__ void __launch_bounds__(GEMM_THREADS) linear_simt_kernel(const float* __restrict__ X, int64_t ldx,
                                                                  const float* __restrict__ W, int64_t ldw,
                                                                  const float* __restrict__ bias,
                                                                  const float* __restrict__ R, int64_t ldr,
                                                                  float* __restrict__ Y, int64_t ldy, int64_t n_rows,
                                                                  int K, int N, int relu_in, int relu_out, int x_vec,
                                                                  int w_vec, int y_vec) {
    __shared__ __align__(16) float As[2][BK][BM + PAD];
    __shared__ __align__(16) float Bs[2][BK][BN + PAD];

    const int tid = threadIdx.x;
    const int64_t m0 = (int64_t)blockIdx.y * BM;
    const int n0 = blockIdx.x * BN;
    const int lrow = tid & 127;          // tile row this thread stages
    const int lk = (tid >> 7) * 8;       // k offset inside the slab (0 or 8)
    const int tx = tid & 15, ty = tid >> 4;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;

    float ra[8], rb[8];
    const int n_slabs = (K + BK - 1) / BK;
    load8(X, ldx, m0 + lrow, n_rows, lk, K, x_vec, relu_in, ra);
    load8(W, ldw, n0 + lrow, N, lk, K, w_vec, 0, rb);
#pragma unroll
    for (int i = 0; i < 8; ++i) { As[0][lk + i][lrow] = ra[i]; Bs[0][lk + i][lrow] = rb[i]; }
    __syncthreads();

    for (int s = 0; s < n_slabs; ++s) {
        const int cur = s & 1;
        if (s + 1 < n_slabs) {
            load8(X, ldx, m0 + lrow, n_rows, (s + 1) * BK + lk, K, x_vec, relu_in, ra);
            load8(W, ldw, n0 + lrow, N, (s + 1) * BK + lk, K, w_vec, 0, rb);
        }
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][k][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (s + 1 < n_slabs) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { As[cur ^ 1][lk + i][lrow] = ra[i]; Bs[cur ^ 1][lk + i][lrow] = rb[i]; }
        }
        __syncthreads();
    }

    // epilogue: bias, activation, residual, store
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t row = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (row >= n_rows) continue;
#pragma unroll
        for (int hj = 0; hj < 2; ++hj) {
            const int col = n0 + hj * 64 + tx * 4;
            if (col >= N) continue;
            float o[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float v = acc[i][hj * 4 + j];
                if (col + j < N) {
                    if (bias) v += __ldg(bias + col + j);
                    if (relu_out) v = nfk_act(relu_out, v);
                    if (R) v += R[row * ldr + col + j];
                }
                o[j] = v;
            }
            if (y_vec && col + 3 < N) {
                *reinterpret_cast<float4*>(Y + row * ldy + col) = make_float4(o[0], o[1], o[2], o[3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (col + j < N) Y[row * ldy + col + j] = o[j];
            }
        }
    }
}

int linear_simt(const float* X, int64_t ldx, const float* W, int64_t ldw, const float* bias, const float* R, int64_t ldr,
                float* Y, int64_t ldy, int64_t n_rows, int K, int N, int relu_in, int relu_out, cudaStream_t st) {
    const int x_vec = aligned16(X) && (ldx % 4 == 0);
    const int w_vec = aligned16(W) && (ldw % 4 == 0);
    const int y_vec = aligned16(Y) && (ldy % 4 == 0);
    const int64_t row_tiles = (n_rows + BM - 1) / BM;
    const int col_tiles = (N + BN - 1) / BN;
    // gridDim.y is limited to 65535: loop over row super-blocks if needed
    for (int64_t t0 = 0; t0 < row_tiles; t0 += 65535) {
        const int64_t nt = row_tiles - t0 < 65535 ? row_tiles - t0 : 65535;
        const int64_t r0 = t0 * BM;
        dim3 grid((unsigned)col_tiles, (unsigned)nt);
        linear_simt_kernel<<<grid, GEMM_THREADS, 0, st>>>(X + r0 * ldx, ldx, W, ldw, bias, R ? R + r0 * ldr : nullptr, ldr,
                                                          Y + r0 * ldy, ldy, n_rows - r0, K, N, relu_in, relu_out, x_vec,
                                                          w_vec, y_vec);
        int rc = check_launch("linear_simt_kernel");
        if (rc) return rc;
    }
    return NFK_OK;
}

}  // namespace nfk

extern "C" int nfk_linear(const float* X, int64_t ldx, const float* W, int64_t ldw, const float* bias, const float* R,
                          int64_t ldr, float* Y, int64_t ldy, int64_t n_rows, int32_t in_features, int32_t out_features,
                          int relu_in, int relu_out, void* stream) {
    NFK_REQUIRE(n_rows >= 0 && in_features >= 1 && out_features >= 1, "bad sizes n=%lld in=%d out=%d", (long long)n_rows,
                in_features, out_features);
    NFK_REQUIRE(nfk::act_valid(relu_in) && nfk::act_valid(relu_out), "unknown activation code (relu_in=%d, relu_out=%d)", relu_in, relu_out);
    if (n_rows == 0) return NFK_OK;
    NFK_REQUIRE(X && W && Y, "NULL pointer");
    NFK_REQUIRE(ldx >= in_features && ldw >= in_features && ldy >= out_features, "row stride smaller than row length");
    NFK_REQUIRE(!R || ldr >= out_features, "residual row stride smaller than row length");
    NFK_REQUIRE(X != Y, "Y must not alias X");
    return nfk::linear_simt(X, ldx, W, ldw, bias, R, ldr, Y, ldy, n_rows, in_features, out_features, relu_in, relu_out,
                            (cudaStream_t)stream);
}
