// fsb200 — FP8 training GEMM and its quantiser for sm_90a: the layer projections of a LLaMA, BERT, MegatronBERT, mT5 or
// GPT-2 model built with fp8=True.
// The recipe (include/fsb200.h): activations and weights e4m3, gradients e5m2, one power-of-two scale per tensor computed
// just in time from the tensor's amax, fp32 accumulation, bf16 outputs.
//
// fsb_fp8_quantize: two launches. (1) amax = max |x| as the maximum of the bf16 magnitude bits (so a NaN, whose magnitude
// bits exceed those of inf, wins), one atomicMax per block into the caller's fp32 scalar. (2) Every block derives the scale
// from amax, casts a 64 x 64 tile (round to nearest even, saturating) and writes its row-major codes directly and its
// transposed codes through a shared-memory tile.
//
// fsb_gemm_fp8: D[m, n] (+)= bf16(sum_k A[m, k] B[n, k] * a_scale_inv * b_scale_inv), both operands K-major FP8 codes.
//   * Persistent, warp-specialised like gemm.cu (TmaRing, tile_coords, the 128B-swizzled TMA-store epilogue): 384 threads,
//     warpgroup 0 = TMA producer, warpgroups 1-2 = consumers, each owning 64 rows of the 128 x 128 tile.
//   * A stage is one 128-deep k-block: a 128 x 128-byte A box and a 128 x 128-byte B box, 128B-swizzled; a k32 FP8 step spans
//     the same 32 bytes as a bf16 k16 step, so the descriptors are gemm.cu's K-major ones.
//   * Promotion: the four m64n128k32 wgmmas of a k-block write a fresh partial sum, which is added into a separate fp32
//     accumulator once they retire (the tensor cores keep fewer than fp32's bits while they accumulate FP8 products). 64 + 64
//     accumulator registers per thread.
//   * Epilogue: acc * a_scale_inv * b_scale_inv (the scales read from device memory: a captured graph stays valid), then,
//     in the kEpi instantiations only, + bias[n] -> aux = bf16(that value) -> GELU (gemm_epilogue.cuh, gemm.cu's device code),
//     plus the old D in fp32 when accumulating, rounded once to bf16, staged in 64-row x 64-column sub-tiles and stored by
//     TMA, which clips ragged m / n edges; aux leaves through the same staging buffers as a second store per sub-tile. The
//     plain instantiations (no bias, aux or activation) are the ones LLaMA runs and carry none of that code. No split-K:
//     results are deterministic.
// fsb_gemm_fp8_t: the same kernel with the kT flag, D[n, m] = the transpose of fsb_gemm_fp8's D. A GPT-2 Conv1D weight is
//   stored [in, out], so its gradient x^T dy must land [in, out]; both FP8 wgmma operands are K-major, which makes the pair
//   the kernel takes, (e5m2, e4m3), compute dy^T x = dW^T. The kT epilogue stages each 64 x 64 sub-tile transposed (stmatrix
//   .trans into the same 128B-swizzled buffers) and TMA-stores it at swapped coordinates; main loop, producer and scales are
//   shared, so the values are fsb_gemm_fp8's bit for bit.
#include "gemm_epilogue.cuh"
#include "host_common.h"
#include "ptx.cuh"

namespace fsb {

constexpr int F8_BM = 128, F8_BN = 128, F8_BK = 128;   // BK: k per stage = one 128-byte swizzle line of FP8 codes per row
constexpr int F8_THREADS = 384;
constexpr int F8_TILE = 64;                            // quantiser tile: 64 rows x 64 columns

struct F8Smem {
  static constexpr int A_BYTES = F8_BM * F8_BK;
  static constexpr int B_BYTES = F8_BN * F8_BK;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = 6;
  static constexpr int EPI_BUF_BYTES = 64 * 128;   // one 64-row x 64-column bf16 sub-tile
  static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = EPI_OFFSET + 2 /*warpgroups*/ * 2 /*buffers*/ * EPI_BUF_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8 + 1024 /*align slack*/;
  static_assert(TOTAL <= kSmemOptIn, "exceeds the 227 KB of shared memory a block can opt into on sm_90");
};

struct F8Params {
  __nv_bfloat16* D;
  const float* a_sinv;
  const float* b_sinv;
  int64_t ldd;
  int M, N, K;
  int accumulate;
  int tiles_m, tiles_n, group_m;
  // read by the kEpi instantiations only (appended, so the plain ones see the parameter block they always had)
  const __nv_bfloat16* bias;   // [N] or null
  int epilogue;                // fsb_gemm_epilogue
  int has_aux;                 // tmAux is valid
};

// kEpi: bias / GELU / aux in the epilogue. tmAux is the last parameter so that the plain kernels' parameter offsets are
// unchanged. kT: D is stored transposed, D[n, m] (fsb_gemm_fp8_t; plain epilogue only): each 64 x 64 sub-tile is staged
// transposed by stmatrix .trans and TMA-stored at swapped coordinates, and the old D of `accumulate` is read at D[col][row].
template <bool kE5M2A, bool kEpi, bool kT = false>
__global__ void __launch_bounds__(F8_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmD, const F8Params p, const __grid_constant__ CUtensorMap tmAux) {
  using S = F8Smem;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  TmaRing<S::STAGES> ring(reinterpret_cast<uint64_t*>(smem + S::BAR_OFFSET));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.tiles_m * p.tiles_n;
  const int num_kb = (p.K + F8_BK - 1) / F8_BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    ring.init();
    fence_barrier_init();
  }
  if (threadIdx.x == 128) {
    tma_prefetch_desc(&tmD);
    if constexpr (kEpi) {
      if (p.has_aux) tma_prefetch_desc(&tmAux);
    }
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    reg_dec<40>();
    if (threadIdx.x == 0) {
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int b, m_idx, n_idx;
        tile_coords(t, p.tiles_m, p.tiles_n, p.group_m, b, m_idx, n_idx);
        for (int kb = 0; kb < num_kb; ++kb) {
          ring.acquire();
          uint8_t* sa = smem + ring.stage * S::STAGE_BYTES;
          uint64_t* bar = ring.expect(S::STAGE_BYTES);
          tma_load_2d(sa, &tmA, bar, kb * F8_BK, m_idx * F8_BM);
          tma_load_2d(sa + S::A_BYTES, &tmB, bar, kb * F8_BK, n_idx * F8_BN);
          ring.advance();
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====================
    reg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int wl = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    const uint64_t dsc_a = make_smem_desc_sw128(smem_u32(smem) + wg * (64 * 128), 0, 1024);
    const uint64_t dsc_b = make_smem_desc_sw128(smem_u32(smem) + S::A_BYTES, 0, 1024);
    uint8_t* const epi_buf = smem + S::EPI_OFFSET + wg * (2 * S::EPI_BUF_BYTES);
    uint32_t n_stored = 0;
    float acc[64], part[64];
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int b, m_idx, n_idx;
      tile_coords(t, p.tiles_m, p.tiles_n, p.group_m, b, m_idx, n_idx);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        ring.wait();
        const uint64_t so = uint64_t(ring.stage) * (S::STAGE_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < F8_BK / 32; ++k)
          wgmma_ss_n128_f8<kE5M2A>(part, dsc_a + so + ((k * 32) >> 4), dsc_b + so + ((k * 32) >> 4), k != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(part);
        ring.release(lane);
        ring.advance();
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] += part[i];   // promotion into the fp32 accumulator, once per 128 k
      }

      // ---- epilogue: accumulator j covers columns 8 (j / 4) + 2 (lane % 4) + (j & 1), rows r and r + 8 (r = 16 wl + lane / 4)
      const float sa = __ldg(p.a_sinv), sb = __ldg(p.b_sinv);
      const int r = wl * 16 + (lane >> 2);
      const int m0 = m_idx * F8_BM + wg * 64, n0 = n_idx * F8_BN;
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = acc[i] * sa * sb;
      if constexpr (kEpi) {
        // bias (0 without one, as gemm.cu: results do not depend on whether a bias was passed)
#pragma unroll
        for (int j = 0; j < F8_BN / 8; ++j) {
          const int col = n0 + 8 * j + 2 * (lane & 3);
          float bv0 = 0.f, bv1 = 0.f;
          if (p.bias != nullptr && col < p.N) {   // N % 8 == 0: col < N implies col + 1 < N
            bv0 = __bfloat162float(__ldg(p.bias + col));
            bv1 = __bfloat162float(__ldg(p.bias + col + 1));
          }
          acc[4 * j] += bv0; acc[4 * j + 1] += bv1; acc[4 * j + 2] += bv0; acc[4 * j + 3] += bv1;
        }
      }
#pragma unroll
      for (int g = 0; g < F8_BN / 64; ++g) {
        if constexpr (kEpi) {
          // pre-activation copy (bf16), through the staging buffers as D below. Written out rather than shared with D's
          // store through a lambda: a lambda capturing these locals, even one the plain kernels never call, changed their
          // instruction schedule.
          if (p.has_aux) {
            uint8_t* buf = epi_buf + (n_stored & 1) * S::EPI_BUF_BYTES;
            if (leader) tma_store_wait_read<1>();
            bar_sync(1 + wg, 128);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int j = 8 * g + jj;
                *reinterpret_cast<uint32_t*>(buf + swz128(r + 8 * h, 16 * jj + 4 * (lane & 3))) =
                    pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
              }
            fence_proxy_async();
            bar_sync(1 + wg, 128);
            if (leader) {
              tma_store_2d(&tmAux, buf, n0 + 64 * g, m0);
              tma_store_commit();
            }
            ++n_stored;
          }
#pragma unroll
          for (int i = 32 * g; i < 32 * g + 32; ++i) {
            if (p.epilogue == FSB_EPI_GELU_TANH) acc[i] = gelu_tanh_f(acc[i]);
            else if (p.epilogue == FSB_EPI_GELU_ERF) acc[i] = gelu_erf_f(acc[i]);
          }
        }
        if (p.accumulate) {   // D += result: fp32 sum with the old value, rounded once
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * g + jj;
            const int col = n0 + 8 * j + 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = m0 + r + 8 * h;
              if constexpr (kT) {   // element (row, col) is D[col][row]; any N, so col + 1 is bounded on its own
                if (row >= p.M) continue;
                if (col < p.N) acc[4 * j + 2 * h] += __bfloat162float(p.D[int64_t(col) * p.ldd + row]);
                if (col + 1 < p.N) acc[4 * j + 2 * h + 1] += __bfloat162float(p.D[int64_t(col + 1) * p.ldd + row]);
              } else {
                if (row >= p.M || col >= p.N) continue;   // N % 8 == 0: col < N implies col + 1 < N
                const uint32_t q = *reinterpret_cast<const uint32_t*>(p.D + int64_t(row) * p.ldd + col);
                acc[4 * j + 2 * h] += bf16lo(q);
                acc[4 * j + 2 * h + 1] += bf16hi(q);
              }
            }
          }
        }
        uint8_t* buf = epi_buf + (n_stored & 1) * S::EPI_BUF_BYTES;
        if (leader) tma_store_wait_read<1>();   // the store that last used this buffer has read it out
        bar_sync(1 + wg, 128);
        if constexpr (kT) {
          // the sub-tile's column c (of 64) becomes buffer row c: 128 bytes = the warpgroup's 64 rows. One stmatrix per two
          // 8-column groups: matrix i = (group jj + i / 2, rows r0 + 8 (i % 2)), r0 = 16 wl; lane 8 i + c addresses its row c.
          const int mi = lane >> 3;
#pragma unroll
          for (int jj = 0; jj < 8; jj += 2) {
            const int j = 8 * g + jj;
            stmatrix_x4_trans(smem_u32(buf + swz128(8 * (jj + (mi >> 1)) + (lane & 7), 32 * wl + 16 * (mi & 1))),
                              pack_bf16x2(acc[4 * j], acc[4 * j + 1]), pack_bf16x2(acc[4 * j + 2], acc[4 * j + 3]),
                              pack_bf16x2(acc[4 * j + 4], acc[4 * j + 5]), pack_bf16x2(acc[4 * j + 6], acc[4 * j + 7]));
          }
        } else {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int j = 8 * g + jj;
              *reinterpret_cast<uint32_t*>(buf + swz128(r + 8 * h, 16 * jj + 4 * (lane & 3))) =
                  pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        }
        fence_proxy_async();
        bar_sync(1 + wg, 128);
        if (leader) {
          if constexpr (kT) tma_store_2d(&tmD, buf, m0, n0 + 64 * g);
          else tma_store_2d(&tmD, buf, n0 + 64 * g, m0);
          tma_store_commit();
        }
        ++n_stored;
      }
    }
    if (leader) tma_store_wait<0>();
  }
}

// ---- quantiser ------------------------------------------------------------------------------------------------------------
// amax bits (fp32) = max over the tile of the bf16 magnitude bits << 16
__global__ void fp8_amax_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols,
                                unsigned* __restrict__ amax_bits) {
  const int64_t c8 = cols / 8, total = rows * c8;
  uint32_t m2 = 0;   // two 16-bit maxima
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / c8, c = (i - r * c8) * 8;
    const uint4 q = *reinterpret_cast<const uint4*>(x + r * ldx + c);
    m2 = __vmaxu2(m2, __vmaxu2(__vmaxu2(q.x & 0x7FFF7FFFu, q.y & 0x7FFF7FFFu), __vmaxu2(q.z & 0x7FFF7FFFu, q.w & 0x7FFF7FFFu)));
  }
  uint32_t m = max(m2 & 0xFFFFu, m2 >> 16);
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ uint32_t red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0u;
    m = __reduce_max_sync(0xffffffffu, m);
    if (threadIdx.x == 0 && m != 0) atomicMax(amax_bits, m << 16);
  }
}

// scale = 2^e, e = floor(log2(fmax / amax)) clamped to [-126, 126], fmax = 1.75 * 2^kEmax (448 for e4m3, 57344 for e5m2).
// With amax = m * 2^(ea - 1), m in [1, 2): fmax / amax = (1.75 / m) 2^(kEmax - ea + 1), and 1.75 / m >= 1 iff m <= 1.75.
// amax == 0: scale = 1. amax not finite: scale = 1 and scale_inv = NaN.
__device__ __forceinline__ void fp8_scale(float amax, int kEmax, float& scale, float& scale_inv) {
  if (!(amax <= 3.402823466e38f)) {
    scale = 1.f;
    scale_inv = __int_as_float(0x7FC00000);
    return;
  }
  int e = 0;
  if (amax > 0.f) {
    int ea;
    const float m = 2.f * frexpf(amax, &ea);
    e = kEmax - (ea - 1) - (m > 1.75f ? 1 : 0);
    e = min(max(e, -126), 126);
  }
  scale = ldexpf(1.f, e);
  scale_inv = ldexpf(1.f, -e);
}

template <bool kE5M2>
__device__ __forceinline__ uint32_t f8x2(float lo, float hi) {   // lo -> byte 0, hi -> byte 1
  uint16_t r;
  if constexpr (kE5M2) asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

template <bool kE5M2>
__global__ void __launch_bounds__(256)
fp8_cast_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, uint8_t* __restrict__ y,
                uint8_t* __restrict__ yt, float* __restrict__ scale_inv, const float* __restrict__ amax) {
  __shared__ __align__(16) uint8_t tile[F8_TILE][F8_TILE + 16];
  float scale, sinv;
  fp8_scale(*amax, kE5M2 ? 15 : 8, scale, sinv);
  if (scale_inv != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *scale_inv = sinv;
  const int64_t r0 = int64_t(blockIdx.y) * F8_TILE, c0 = int64_t(blockIdx.x) * F8_TILE;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int idx = threadIdx.x + 256 * j;
    const int lr = idx >> 3, lc = (idx & 7) * 8;
    const int64_t r = r0 + lr, c = c0 + lc;
    if (r < rows && c < cols) {
      float v[8];
      unpack8(*reinterpret_cast<const uint4*>(x + r * ldx + c), v);
      uint2 q;
      q.x = f8x2<kE5M2>(v[0] * scale, v[1] * scale) | (f8x2<kE5M2>(v[2] * scale, v[3] * scale) << 16);
      q.y = f8x2<kE5M2>(v[4] * scale, v[5] * scale) | (f8x2<kE5M2>(v[6] * scale, v[7] * scale) << 16);
      if (y != nullptr) *reinterpret_cast<uint2*>(y + r * cols + c) = q;
      *reinterpret_cast<uint2*>(&tile[lr][lc]) = q;
    }
  }
  if (yt == nullptr) return;
  __syncthreads();
  // yt row c0 + lc, bytes [16 part, 16 part + 16) of the tile's rows (rows % 16 == 0: a chunk is all in or all out)
  const int lc = threadIdx.x >> 2, part = threadIdx.x & 3;
  const int64_t c = c0 + lc, r = r0 + 16 * part;
  if (c < cols && r < rows) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int b = 16 * part + 4 * i;
      w[i] = uint32_t(tile[b][lc]) | (uint32_t(tile[b + 1][lc]) << 8) | (uint32_t(tile[b + 2][lc]) << 16) |
             (uint32_t(tile[b + 3][lc]) << 24);
    }
    *reinterpret_cast<uint4*>(yt + c * rows + r) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

template <bool kE5M2A, bool kEpi, bool kT = false>
static int launch_gemm_fp8(int grid, const F8Params& p, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD,
                           const CUtensorMap& tmAux, cudaStream_t stream) {
  if (int rc = ensure_smem<gemm_fp8_kernel<kE5M2A, kEpi, kT>>(F8Smem::TOTAL, "gemm_fp8")) return rc;
  gemm_fp8_kernel<kE5M2A, kEpi, kT><<<grid, F8_THREADS, F8Smem::TOTAL, stream>>>(tmA, tmB, tmD, p, tmAux);
  return FSB_OK;
}

// The tensor maps, tile schedule and launch of fsb_gemm_fp8 (transposed = false: D [m, n]) and fsb_gemm_fp8_t (D [n, m]),
// after each entry's own checks.
static int run_gemm_fp8(bool transposed, int64_t m, int64_t n, int64_t k, const void* a, int a_fmt, const float* a_scale_inv,
                        const void* b, const float* b_scale_inv, void* d, int64_t ldd, const void* bias, int epilogue,
                        int accumulate, void* aux, int64_t ldaux, cudaStream_t stream) {
  const bool epi = bias != nullptr || aux != nullptr || epilogue != FSB_EPI_NONE;
  CUtensorMap tmA, tmB, tmD, tmAux;
  {
    uint64_t dims[2] = {uint64_t(k), uint64_t(m)};
    uint64_t strides[1] = {uint64_t(k)};
    uint32_t box[2] = {uint32_t(F8_BK), uint32_t(F8_BM)};
    if (int rc = make_tmap_u8(&tmA, a, 2, dims, strides, box)) return rc;
  }
  {
    uint64_t dims[2] = {uint64_t(k), uint64_t(n)};
    uint64_t strides[1] = {uint64_t(k)};
    uint32_t box[2] = {uint32_t(F8_BK), uint32_t(F8_BN)};
    if (int rc = make_tmap_u8(&tmB, b, 2, dims, strides, box)) return rc;
  }
  {
    uint64_t dims[2] = {uint64_t(transposed ? m : n), uint64_t(transposed ? n : m)};
    uint64_t strides[1] = {uint64_t(ldd) * 2};
    uint32_t box[2] = {64, 64};
    if (int rc = make_tmap_bf16(&tmD, d, 2, dims, strides, box)) return rc;
  }
  tmAux = tmD;   // never read without aux
  if (aux != nullptr) {
    uint64_t dims[2] = {uint64_t(n), uint64_t(m)};
    uint64_t strides[1] = {uint64_t(ldaux) * 2};
    uint32_t box[2] = {64, 64};
    if (int rc = make_tmap_bf16(&tmAux, aux, 2, dims, strides, box)) return rc;
  }
  F8Params p;
  p.D = static_cast<__nv_bfloat16*>(d);
  p.a_sinv = a_scale_inv; p.b_sinv = b_scale_inv;
  p.ldd = ldd;
  p.M = int(m); p.N = int(n); p.K = int(k);
  p.accumulate = accumulate;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.epilogue = epilogue;
  p.has_aux = aux != nullptr;
  p.tiles_m = int((m + F8_BM - 1) / F8_BM);
  p.tiles_n = int((n + F8_BN - 1) / F8_BN);
  // rasterisation groups as gemm.cu's 128-wide tiles: 12 m-tiles, more while their A panels (128 x k bytes) fit ~32 MB of L2
  {
    int64_t gm = (int64_t(32) << 20) / (int64_t(F8_BM) * k);
    p.group_m = int(gm < 12 ? 12 : (gm > 64 ? 64 : gm));
  }
  const int num_tiles = p.tiles_m * p.tiles_n;
  const int grid = num_tiles < gemm_sms() ? num_tiles : gemm_sms();
  int rc;
  if (transposed) rc = launch_gemm_fp8<true, false, true>(grid, p, tmA, tmB, tmD, tmAux, stream);
  else if (a_fmt == FSB_FP8_E5M2) rc = epi ? launch_gemm_fp8<true, true>(grid, p, tmA, tmB, tmD, tmAux, stream)
                                           : launch_gemm_fp8<true, false>(grid, p, tmA, tmB, tmD, tmAux, stream);
  else rc = epi ? launch_gemm_fp8<false, true>(grid, p, tmA, tmB, tmD, tmAux, stream)
                : launch_gemm_fp8<false, false>(grid, p, tmA, tmB, tmD, tmAux, stream);
  if (rc) return rc;
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

}  // namespace fsb

using namespace fsb;

extern "C" int fsb_fp8_quantize(const void* x, int64_t ldx, int64_t rows, int64_t cols, int fmt, void* y, void* yt,
                                float* scale_inv, float* amax, fsb_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FSB_REQUIRE(rows > 0 && cols > 0, "fp8_quantize: non-positive dims rows=%ld cols=%ld", (long)rows, (long)cols);
  FSB_REQUIRE(rows % 16 == 0 && cols % 16 == 0, "fp8_quantize: rows=%ld and cols=%ld must be multiples of 16", (long)rows,
              (long)cols);
  FSB_REQUIRE(rows < (int64_t(1) << 31) && cols < (int64_t(1) << 31) && (rows + F8_TILE - 1) / F8_TILE <= 65535,
              "fp8_quantize: rows=%ld or cols=%ld too large", (long)rows, (long)cols);
  FSB_REQUIRE(fmt == FSB_FP8_E4M3 || fmt == FSB_FP8_E5M2, "fp8_quantize: bad format %d", fmt);
  FSB_REQUIRE(ldx >= cols && ldx % 8 == 0, "fp8_quantize: ldx=%ld must be >= cols and a multiple of 8", (long)ldx);
  FSB_REQUIRE(x && amax, "fp8_quantize: null x or amax");
  FSB_REQUIRE(aligned16(x) && (y == nullptr || aligned16(y)) && (yt == nullptr || aligned16(yt)) &&
                  (reinterpret_cast<uintptr_t>(amax) & 3) == 0 && (reinterpret_cast<uintptr_t>(scale_inv) & 3) == 0,
              "fp8_quantize: x, y and yt must be 16-byte aligned, amax and scale_inv 4-byte aligned");
  if (const cudaError_t e = cudaMemsetAsync(amax, 0, sizeof(float), stream)) {
    set_error("fp8_quantize: clearing amax failed: %s", cudaGetErrorString(e));
    return FSB_ERR_CUDA;
  }
  const int64_t work = rows * (cols / 8);
  const int64_t cap = 4 * int64_t(num_sms());
  const unsigned blocks = unsigned(work / 256 + 1 < cap ? work / 256 + 1 : cap);
  fp8_amax_kernel<<<blocks, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), ldx, rows, cols,
                                              reinterpret_cast<unsigned*>(amax));
  FSB_CUDA_LAUNCH_CHECK();
  const dim3 grid(unsigned((cols + F8_TILE - 1) / F8_TILE), unsigned((rows + F8_TILE - 1) / F8_TILE));
  auto* xb = static_cast<const __nv_bfloat16*>(x);
  auto* yb = static_cast<uint8_t*>(y);
  auto* ytb = static_cast<uint8_t*>(yt);
  if (fmt == FSB_FP8_E5M2) fp8_cast_kernel<true><<<grid, 256, 0, stream>>>(xb, ldx, rows, cols, yb, ytb, scale_inv, amax);
  else fp8_cast_kernel<false><<<grid, 256, 0, stream>>>(xb, ldx, rows, cols, yb, ytb, scale_inv, amax);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

extern "C" int fsb_gemm_fp8(int64_t m, int64_t n, int64_t k, const void* a, int a_fmt, const float* a_scale_inv,
                            const void* b, int b_fmt, const float* b_scale_inv, void* d, int64_t ldd, const void* bias,
                            int epilogue, int accumulate, void* aux, int64_t ldaux, fsb_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FSB_REQUIRE(m > 0 && n > 0 && k > 0, "gemm_fp8: non-positive dims m=%ld n=%ld k=%ld", (long)m, (long)n, (long)k);
  FSB_REQUIRE(m < (1 << 30) && n < (1 << 30) && k < (1 << 30), "gemm_fp8: dims too large");
  FSB_REQUIRE(k % 16 == 0, "gemm_fp8: k=%ld must be a multiple of 16", (long)k);
  FSB_REQUIRE(n % 8 == 0, "gemm_fp8: n=%ld must be a multiple of 8", (long)n);
  FSB_REQUIRE(b_fmt == FSB_FP8_E4M3 && (a_fmt == FSB_FP8_E4M3 || a_fmt == FSB_FP8_E5M2),
              "gemm_fp8: format pair (a %d, b %d) unsupported: (e4m3, e4m3) or (e5m2, e4m3)", a_fmt, b_fmt);
  FSB_REQUIRE(a && b && d && a_scale_inv && b_scale_inv, "gemm_fp8: null operand");
  FSB_REQUIRE(aligned16(a) && aligned16(b) && aligned16(d), "gemm_fp8: a, b and d must be 16-byte aligned");
  FSB_REQUIRE((reinterpret_cast<uintptr_t>(a_scale_inv) & 3) == 0 && (reinterpret_cast<uintptr_t>(b_scale_inv) & 3) == 0,
              "gemm_fp8: scale_inv pointers must be 4-byte aligned");
  FSB_REQUIRE(ldd >= n && ldd % 8 == 0, "gemm_fp8: ldd=%ld must be >= n and a multiple of 8", (long)ldd);
  FSB_REQUIRE(epilogue >= FSB_EPI_NONE && epilogue <= FSB_EPI_GELU_ERF, "gemm_fp8: bad epilogue %d", epilogue);
  FSB_REQUIRE(bias == nullptr || aligned16(bias), "gemm_fp8: bias must be 16-byte aligned");
  FSB_REQUIRE(aux == nullptr || (aligned16(aux) && ldaux >= n && ldaux % 8 == 0),
              "gemm_fp8: aux must be 16-byte aligned with ldaux=%ld >= n and a multiple of 8", (long)ldaux);
  return run_gemm_fp8(false, m, n, k, a, a_fmt, a_scale_inv, b, b_scale_inv, d, ldd, bias, epilogue, accumulate, aux, ldaux,
                      stream);
}

extern "C" int fsb_gemm_fp8_t(int64_t m, int64_t n, int64_t k, const void* a, int a_fmt, const float* a_scale_inv,
                              const void* b, int b_fmt, const float* b_scale_inv, void* d, int64_t ldd, const void* bias,
                              int epilogue, int accumulate, void* aux, int64_t ldaux, fsb_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FSB_REQUIRE(m > 0 && n > 0 && k > 0, "gemm_fp8_t: non-positive dims m=%ld n=%ld k=%ld", (long)m, (long)n, (long)k);
  FSB_REQUIRE(m < (1 << 30) && n < (1 << 30) && k < (1 << 30), "gemm_fp8_t: dims too large");
  FSB_REQUIRE(k % 16 == 0, "gemm_fp8_t: k=%ld must be a multiple of 16", (long)k);
  FSB_REQUIRE(m % 8 == 0, "gemm_fp8_t: m=%ld must be a multiple of 8 (D^T rows of m bf16 values need 16-byte strides)",
              (long)m);
  FSB_REQUIRE(a_fmt == FSB_FP8_E5M2 && b_fmt == FSB_FP8_E4M3,
              "gemm_fp8_t: format pair (a %d, b %d) unsupported: only (e5m2, e4m3)", a_fmt, b_fmt);
  FSB_REQUIRE(bias == nullptr && aux == nullptr && epilogue == FSB_EPI_NONE,
              "gemm_fp8_t: no bias, aux or epilogue (got bias %s, aux %s, epilogue %d)", bias ? "set" : "NULL",
              aux ? "set" : "NULL", epilogue);
  FSB_REQUIRE(a && b && d && a_scale_inv && b_scale_inv, "gemm_fp8_t: null operand");
  FSB_REQUIRE(aligned16(a) && aligned16(b) && aligned16(d), "gemm_fp8_t: a, b and d must be 16-byte aligned");
  FSB_REQUIRE((reinterpret_cast<uintptr_t>(a_scale_inv) & 3) == 0 && (reinterpret_cast<uintptr_t>(b_scale_inv) & 3) == 0,
              "gemm_fp8_t: scale_inv pointers must be 4-byte aligned");
  FSB_REQUIRE(ldd >= m && ldd % 8 == 0, "gemm_fp8_t: ldd=%ld must be >= m and a multiple of 8", (long)ldd);
  (void)ldaux;
  return run_gemm_fp8(true, m, n, k, a, a_fmt, a_scale_inv, b, b_scale_inv, d, ldd, nullptr, FSB_EPI_NONE, accumulate,
                      nullptr, 0, stream);
}
