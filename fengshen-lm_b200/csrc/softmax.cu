// fsb200 — the reference's two in-tree CUDA ops, re-designed for sm_90a (HBM-bound row softmax):
//   scaled_masked_softmax_cuda.{forward,backward}              fused_kernels/scaled_masked_softmax.h:117-335
//       y = softmax(mask ? -10000 : scale * x) over the last dim;  x [b, np, sq, sk], mask uint8 [b|1, 1, sq, sk]
//       dx = scale * (dy*y - y * sum(dy*y)), written IN PLACE over dy (scaled_masked_softmax_cuda.cu:95-105)
//   scaled_upper_triang_masked_softmax_cuda.{forward,backward} fused_kernels/scaled_upper_triang_masked_softmax.h:143-363
//       causal variant on [attn_batches, s, s]: row r normalises its first r+1 elements, zeros above the diagonal.
// The reference builds these for sm_70/sm_80 with one template instance per log2(sk) (12-way switch, silently doing
// nothing for other sizes, scaled_masked_softmax.h:448). Here: one warp per row, the row in registers as 16-byte
// vectors (sk % 8 == 0, sk <= 4096), fp32 statistics via shuffles, grid = rows / 4 warps. Algorithmic traffic:
// forward 2 B read + 1 B mask + 2 B write per element; backward 4 B read + 2 B write.
#include "host_common.h"
#include "ptx.cuh"

namespace fsb {

constexpr int SM_WARPS = 4;

__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// kCausal: rows are [attn_batches, s, s]; valid length of row r is (r % s) + 1.  Otherwise `mask` (may be null) applies.
template <int VPL, bool kCausal>
__global__ void __launch_bounds__(SM_WARPS * 32) softmax_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                                    const uint8_t* __restrict__ mask,
                                                                    __nv_bfloat16* __restrict__ y, int64_t rows, int sk,
                                                                    int sq, int np, int mask_batches, float scale) {
  const int lane = threadIdx.x & 31;
  const int64_t row = int64_t(blockIdx.x) * SM_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = sk >> 3;
  const int valid = kCausal ? int(row % sq) + 1 : sk;
  // mask row: [b | 1, 1, sq, sk]; row index = ((b * np + h) * sq + q)
  const uint8_t* mrow = nullptr;
  if (!kCausal && mask != nullptr) {
    const int64_t q = row % sq, bh = row / sq, bidx = bh / np;
    mrow = mask + ((mask_batches == 1 ? 0 : bidx) * sq + q) * int64_t(sk);
  }
  float v[VPL][8];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec && (!kCausal || c * 8 < valid)) {
      unpack8(*reinterpret_cast<const uint4*>(x + row * sk + c * 8), v[i]);
      uint2 mk = make_uint2(0, 0);
      if (mrow) mk = *reinterpret_cast<const uint2*>(mrow + c * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool masked = mrow && ((j < 4 ? (mk.x >> (8 * j)) : (mk.y >> (8 * (j - 4)))) & 0xff) == 1;
        float a = masked ? -10000.f : v[i][j] * scale;          // scaled_masked_softmax.h:183
        if (kCausal && c * 8 + j >= valid) a = -INFINITY;
        v[i][j] = a;
        mx = fmaxf(mx, a);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = -INFINITY;
    }
  }
  mx = wmax(mx);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[i][j] = __expf(v[i][j] - mx); sum += v[i][j]; }
  sum = wsum(sum);
  const float inv = 1.f / sum;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = v[i][j] * inv;   // elements above the diagonal: exp(-inf) = 0
      *reinterpret_cast<uint4*>(y + row * sk + c * 8) = pack8(o);
    }
  }
}

template <int VPL, bool kCausal>
__global__ void __launch_bounds__(SM_WARPS * 32) softmax_bwd_kernel(__nv_bfloat16* __restrict__ dy /* in place */,
                                                                    const __nv_bfloat16* __restrict__ y, int64_t rows,
                                                                    int sk, int sq, float scale) {
  const int lane = threadIdx.x & 31;
  const int64_t row = int64_t(blockIdx.x) * SM_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = sk >> 3;
  const int valid = kCausal ? int(row % sq) + 1 : sk;
  float g[VPL][8], p[VPL][8];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec && (!kCausal || c * 8 < valid)) {
      unpack8(*reinterpret_cast<const uint4*>(dy + row * sk + c * 8), g[i]);
      unpack8(*reinterpret_cast<const uint4*>(y + row * sk + c * 8), p[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (kCausal && c * 8 + j >= valid) { g[i][j] = 0.f; p[i][j] = 0.f; }
        dot += g[i][j] * p[i][j];
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) { g[i][j] = 0.f; p[i][j] = 0.f; }
    }
  }
  dot = wsum(dot);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = scale * (g[i][j] * p[i][j] - p[i][j] * dot);   // scaled_masked_softmax.h:318-326
      *reinterpret_cast<uint4*>(dy + row * sk + c * 8) = pack8(o);
    }
  }
}

template <bool kCausal>
static int softmax_fwd(const void* x, const uint8_t* mask, void* y, int64_t rows, int sk, int sq, int np,
                       int mask_batches, float scale, cudaStream_t st) {
  const int vpl = (sk / 8 + 31) / 32;
  const unsigned grid = unsigned((rows + SM_WARPS - 1) / SM_WARPS);
#define L(V)                                                                                                      \
  softmax_fwd_kernel<V, kCausal><<<grid, SM_WARPS * 32, 0, st>>>((const __nv_bfloat16*)x, mask, (__nv_bfloat16*)y, \
                                                                 rows, sk, sq, np, mask_batches, scale)
  if (vpl <= 1) L(1); else if (vpl <= 2) L(2); else if (vpl <= 4) L(4); else if (vpl <= 8) L(8); else L(16);
#undef L
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
template <bool kCausal>
static int softmax_bwd(void* dy, const void* y, int64_t rows, int sk, int sq, float scale, cudaStream_t st) {
  const int vpl = (sk / 8 + 31) / 32;
  const unsigned grid = unsigned((rows + SM_WARPS - 1) / SM_WARPS);
#define L(V) \
  softmax_bwd_kernel<V, kCausal><<<grid, SM_WARPS * 32, 0, st>>>((__nv_bfloat16*)dy, (const __nv_bfloat16*)y, rows, sk, sq, scale)
  if (vpl <= 1) L(1); else if (vpl <= 2) L(2); else if (vpl <= 4) L(4); else if (vpl <= 8) L(8); else L(16);
#undef L
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

}  // namespace fsb

using namespace fsb;

extern "C" int fsb_scaled_masked_softmax_fwd(const void* x, const uint8_t* mask, void* y, int64_t batches,
                                             int64_t attn_heads, int64_t sq, int64_t sk, int64_t mask_batches,
                                             float scale, fsb_stream_t st) {
  FSB_REQUIRE(x && y, "scaled_masked_softmax_fwd: null pointer");
  FSB_REQUIRE(batches > 0 && attn_heads > 0 && sq > 0 && sk > 0 && sk % 8 == 0 && sk <= 4096,
              "scaled_masked_softmax_fwd: sk=%ld must be a multiple of 8 and <= 4096", (long)sk);
  FSB_REQUIRE(mask == nullptr || mask_batches == 1 || mask_batches == batches,
              "scaled_masked_softmax_fwd: mask batch must be 1 or %ld", (long)batches);   // _cuda.cu:46
  FSB_REQUIRE(aligned16(x) && aligned16(y) && (reinterpret_cast<uintptr_t>(mask) & 7) == 0, "scaled_masked_softmax_fwd: alignment");
  return softmax_fwd<false>(x, mask, y, batches * attn_heads * sq, int(sk), int(sq), int(attn_heads), int(mask_batches),
                            scale, (cudaStream_t)st);
}
extern "C" int fsb_scaled_masked_softmax_bwd(void* dy_inplace, const void* y, int64_t rows, int64_t sk, float scale,
                                             fsb_stream_t st) {
  FSB_REQUIRE(dy_inplace && y && rows > 0 && sk > 0 && sk % 8 == 0 && sk <= 4096, "scaled_masked_softmax_bwd: bad args");
  FSB_REQUIRE(aligned16(dy_inplace) && aligned16(y), "scaled_masked_softmax_bwd: alignment");
  return softmax_bwd<false>(dy_inplace, y, rows, int(sk), int(sk), scale, (cudaStream_t)st);
}
extern "C" int fsb_scaled_upper_triang_masked_softmax_fwd(const void* x, void* y, int64_t attn_batches, int64_t seq_len,
                                                          float scale, fsb_stream_t st) {
  FSB_REQUIRE(x && y && attn_batches > 0 && seq_len > 0 && seq_len % 8 == 0 && seq_len <= 4096,
              "scaled_upper_triang_masked_softmax_fwd: seq_len must be a multiple of 8 and <= 4096");
  FSB_REQUIRE(aligned16(x) && aligned16(y), "scaled_upper_triang_masked_softmax_fwd: alignment");
  return softmax_fwd<true>(x, nullptr, y, attn_batches * seq_len, int(seq_len), int(seq_len), 1, 1, scale, (cudaStream_t)st);
}
extern "C" int fsb_scaled_upper_triang_masked_softmax_bwd(void* dy_inplace, const void* y, int64_t attn_batches,
                                                          int64_t seq_len, float scale, fsb_stream_t st) {
  FSB_REQUIRE(dy_inplace && y && attn_batches > 0 && seq_len > 0 && seq_len % 8 == 0 && seq_len <= 4096,
              "scaled_upper_triang_masked_softmax_bwd: bad args");
  FSB_REQUIRE(aligned16(dy_inplace) && aligned16(y), "scaled_upper_triang_masked_softmax_bwd: alignment");
  return softmax_bwd<true>(dy_inplace, y, attn_batches * seq_len, int(seq_len), int(seq_len), scale, (cudaStream_t)st);
}
// get_batch_per_block of the reference (scaled_masked_softmax.h:337-349): rows per 128-thread block of ITS kernel; kept
// because layers/fused_softmax.py:163-170 gates the fused path on `sq % batch_per_block == 0`.
extern "C" int fsb_softmax_get_batch_per_block(int64_t sq, int64_t sk, int64_t batches, int64_t attn_heads) {
  (void)sq; (void)batches; (void)attn_heads;
  int log2_elements = 0;
  while ((int64_t(1) << log2_elements) < sk) ++log2_elements;
  const int next_pow2 = 1 << log2_elements;
  const int warp_size = next_pow2 < 32 ? next_pow2 : 32;
  const int batches_per_warp = next_pow2 <= 128 ? 2 : 1;
  const int warps_per_block = 128 / warp_size;
  return warps_per_block * batches_per_warp;
}
