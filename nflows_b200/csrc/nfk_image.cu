// Image path (SURVEY.md section 8 row f3, BASELINE cfg 5): the per-pixel form of the 4-D transforms.
//
// Inside a native image chain the tensor lives as PIXEL ROWS, [B*H*W, C] fp32 (channels last): ActNorm, OneByOneConvolution and
// the channel-wise RQ coupling of the reference (normalization.py:178-186, conv.py:17-29, coupling.py:280-285) are then exactly
// the 2-D transforms on those rows, and the kernels of the 2-D path run unchanged.  What this file adds is the index shuffling
// around them -- all HBM-bound, one pass each:
//   nchw_to_rows / rows_to_nchw : layout change at the chain's ends (batched 32x32 shared-memory transposes)
//   squeeze_rows                : SqueezeTransform (reshape.py:7-68) on pixel rows, forward and inverse
//   im2col3x3_f16               : the K-major operand of a 3x3 / padding 1 convolution (ConvResidualBlock, resnet.py:103-160)
//                                 from the fp16 pair of its input: [B*H*W, C] -> [B*H*W, 9*C], zero outside the image
//   segment_sum                 : per-pixel log|det| -> per-sample (the reference sums over C, H, W: torchutils.sum_except_batch)
#include "nfk_common.cuh"

#include <cuda_fp16.h>

namespace nfk {

// x: [B, C, P] (P = H*W pixels), rows: [B*P, C].  One 32x32 tile per block, coalesced on both sides.
__global__ void __launch_bounds__(256) nchw_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int c, int p, int to_rows) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    // to_rows: src is [C][P] (inner P), dst is [P][C] (inner C); else the other way round
    const int inner_src = to_rows ? p : c, inner_dst = to_rows ? c : p;
    const int i0 = blockIdx.x * 32, o0 = blockIdx.y * 32;          // i: index along src's inner dim, o: along src's outer dim
    const float* s = src + (int64_t)b * c * p;
    float* d = dst + (int64_t)b * c * p;
    const int outer_src = to_rows ? c : p;
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int o = o0 + r, i = i0 + threadIdx.x;
        if (o < outer_src && i < inner_src) tile[r][threadIdx.x] = s[(int64_t)o * inner_src + i];
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int i = i0 + r, o = o0 + threadIdx.x;                // dst[i][o]
        if (i < inner_src && o < outer_src) d[(int64_t)i * inner_dst + o] = tile[threadIdx.x][r];
    }
}

// forward: out[(b, y', x'), c*4 + dy*2 + dx] = in[(b, 2y'+dy, 2x'+dx), c]   (in: H x W pixels of C channels)
// inverse: out[(b, 2y'+dy, 2x'+dx), c] = in[(b, y', x'), c*4 + dy*2 + dx]   (in: H x W pixels of 4C channels... given as h, w, c of
//          the SQUEEZED side in both directions)
__global__ void __launch_bounds__(256) squeeze_rows_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t n_images,
                                                           int h2, int w2, int c, int inverse) {
    // (h2, w2): squeezed grid, c: channels of the UNSQUEEZED side; one thread per element of the squeezed tensor
    const int c4 = c * 4;
    const int64_t total = n_images * h2 * w2 * c4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(i % c4);
        const int64_t pix = i / c4;
        const int x2 = (int)(pix % w2);
        const int y2 = (int)((pix / w2) % h2);
        const int64_t b = pix / ((int64_t)w2 * h2);
        const int ch = k >> 2, dy = (k >> 1) & 1, dx = k & 1;
        const int64_t big = ((b * (2 * h2) + 2 * y2 + dy) * (2 * w2) + 2 * x2 + dx) * c + ch;
        if (inverse) out[big] = in[i];
        else out[i] = in[big];
    }
}

// One thread per 8 halfs (16 bytes) of the output pair when C % 8 == 0, else per element.
template <int VEC>
__global__ void __launch_bounds__(256) im2col3x3_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, int64_t lds,
                                                        __half* __restrict__ out_hi, __half* __restrict__ out_lo, int64_t ldo,
                                                        int64_t n_images, int h, int w, int c) {
    const int cv = c / VEC;
    const int64_t total = n_images * h * w * 9 * cv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int ch = (int)(i % cv) * VEC;
        const int tap = (int)((i / cv) % 9);
        const int64_t pix = i / ((int64_t)cv * 9);
        const int x = (int)(pix % w);
        const int y = (int)((pix / w) % h);
        const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
        const bool inside = yy >= 0 && yy < h && xx >= 0 && xx < w;
        const int64_t src = (pix + (int64_t)(yy - y) * w + (xx - x)) * lds + ch;
        const int64_t dst = pix * ldo + (int64_t)tap * c + ch;
        if (VEC == 8) {
            uint4 vh = make_uint4(0, 0, 0, 0), vl = make_uint4(0, 0, 0, 0);
            if (inside) {
                vh = *reinterpret_cast<const uint4*>(hi + src);
                vl = *reinterpret_cast<const uint4*>(lo + src);
            }
            *reinterpret_cast<uint4*>(out_hi + dst) = vh;
            *reinterpret_cast<uint4*>(out_lo + dst) = vl;
        } else {
            out_hi[dst] = inside ? hi[src] : __float2half(0.0f);
            out_lo[dst] = inside ? lo[src] : __float2half(0.0f);
        }
    }
}

// out[s] += sum_i v[s * len + i], one warp per segment, fixed order (deterministic)
__global__ void __launch_bounds__(256) segment_sum_kernel(const float* __restrict__ v, float* __restrict__ out, int64_t n_segments, int len) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t s = warp; s < n_segments; s += warps) {
        float acc = 0.0f;
        for (int i = lane; i < len; i += 32) acc += v[s * len + i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) out[s] += acc;
    }
}

static int grid_1d(int64_t work, int threads) {
    int64_t blocks = (work + threads - 1) / threads;
    const int64_t cap = (int64_t)nfk::tc::sm_count() * 16;
    return (int)(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}

}  // namespace nfk

using namespace nfk;

extern "C" int nfk_nchw_to_rows(const float* x, float* rows, int64_t n_images, int32_t channels, int32_t pixels, int to_nchw,
                                void* stream) {
    NFK_REQUIRE(n_images >= 0 && channels >= 1 && pixels >= 1 && n_images < 65536, "bad sizes");
    if (n_images == 0) return NFK_OK;
    NFK_REQUIRE(x && rows, "NULL pointer");
    const int to_rows = to_nchw ? 0 : 1;
    const int inner = to_rows ? pixels : channels, outer = to_rows ? channels : pixels;
    dim3 grid((inner + 31) / 32, (outer + 31) / 32, (unsigned)n_images), block(32, 8);
    NFK_REQUIRE(grid.y < 65536, "image too large for one launch");
    nchw_rows_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, rows, channels, pixels, to_rows);
    return check_launch("nchw_rows_kernel");
}

extern "C" int nfk_squeeze_rows(const float* in, float* out, int64_t n_images, int32_t h2, int32_t w2, int32_t channels, int inverse,
                                void* stream) {
    NFK_REQUIRE(n_images >= 0 && h2 >= 1 && w2 >= 1 && channels >= 1, "bad sizes");
    if (n_images == 0) return NFK_OK;
    NFK_REQUIRE(in && out && in != out, "NULL or aliased pointer");
    squeeze_rows_kernel<<<grid_1d(n_images * h2 * w2 * channels * 4, 256), 256, 0, (cudaStream_t)stream>>>(in, out, n_images, h2, w2,
                                                                                                          channels, inverse);
    return check_launch("squeeze_rows_kernel");
}

extern "C" int nfk_im2col3x3_f16(const void* hi, const void* lo, int64_t lds, void* out_hi, void* out_lo, int64_t ldo, int64_t n_images,
                                 int32_t h, int32_t w, int32_t channels, void* stream) {
    NFK_REQUIRE(n_images >= 0 && h >= 1 && w >= 1 && channels >= 1 && ldo >= 9 * (int64_t)channels && lds >= channels, "bad sizes");
    if (n_images == 0) return NFK_OK;
    NFK_REQUIRE(hi && lo && out_hi && out_lo, "NULL pointer");
    const bool vec = channels % 8 == 0 && lds % 8 == 0 && ldo % 8 == 0 && aligned16(hi) && aligned16(lo) && aligned16(out_hi) &&
                     aligned16(out_lo);
    const int64_t work = n_images * h * w * 9 * (vec ? channels / 8 : channels);
    if (vec)
        im2col3x3_kernel<8><<<grid_1d(work, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)hi, (const __half*)lo, lds, (__half*)out_hi,
                                                                                   (__half*)out_lo, ldo, n_images, h, w, channels);
    else
        im2col3x3_kernel<1><<<grid_1d(work, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)hi, (const __half*)lo, lds, (__half*)out_hi,
                                                                                   (__half*)out_lo, ldo, n_images, h, w, channels);
    return check_launch("im2col3x3_kernel");
}

extern "C" int nfk_segment_sum(const float* values, float* out_accum, int64_t n_segments, int32_t segment_len, void* stream) {
    NFK_REQUIRE(n_segments >= 0 && segment_len >= 1, "bad sizes");
    if (n_segments == 0) return NFK_OK;
    NFK_REQUIRE(values && out_accum, "NULL pointer");
    segment_sum_kernel<<<grid_1d(n_segments * 32, 256), 256, 0, (cudaStream_t)stream>>>(values, out_accum, n_segments, segment_len);
    return check_launch("segment_sum_kernel");
}
