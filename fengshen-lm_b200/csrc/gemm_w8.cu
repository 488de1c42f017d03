// fsb200 — weight-only GEMMs (W8A16, W4A16) and their quantisers for sm_90a: the inference layers behind `load_in_8bit=True`
// and `load_in_4bit=True` (fengshen/examples/ziya_inference/hf_quantizatin_inference.py). The formats (include/fsb200.h):
//   * int8: q int8 [n, k] with one fp32 scale per output channel, s[n] = absmax(W[n, :]) / 127; the GEMM computes
//     D[m, n] = bf16(s[n] * sum_k A[m, k] q[n, k]) with fp32 accumulation.
//   * int4: q in [-7, 7], two per byte, with one bf16 scale per output channel and group of 128 k; the GEMM computes
//     D[m, n] = bf16(sum_k A[m, k] bf16(q[n, k] s[n, k / 128])) with fp32 accumulation.
//
// The operands are swapped against gemm.cu: decode has 1-32 token rows, far below the 64-row minimum of a wgmma A operand, so
// the WEIGHT tile is the A operand and the token tile the B operand (n = 8..128 tokens per tile). One kernel template serves
// both formats; the format decides the weight tile's layout, how a fragment is converted and where the scale is applied.
//   * Roles (384 threads = 3 warpgroups): warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, each owning
//     64 of the tile's 128 weight rows.
//   * Per stage (128 k) the producer loads the tile's 128 weight rows of quantised weights (int8: 128 rows x 128 bytes; int4:
//     64 row pairs x 128 bytes) and two 64-wide bf16 token boxes, all 128B-swizzled; TMA zero-fills token rows at or beyond m
//     and weight rows at or beyond n.
//   * Each consumer thread reads its fragment of the weight tile, converts it to bf16 in registers and issues wgmma in the
//     register-A form against the token tile in shared memory. Two fragment buffers let one stage's conversion overlap the
//     previous stage's MMAs.
//       int8: 2-byte pieces ((row, k..k+1) as the register-A layout places them), converted exactly (every int8 is a bf16).
//       int4: the whole fragment of a k16 step is one 32-bit word: a warp's wgmma rows g and g + 8 are weight rows 2g and
//       2g + 1 of its 16, and one 128-byte line holds a row pair. Each pair of codes becomes bf16(q * s) with the stage's
//       group scale (a stage is one group) before the MMA.
//   * Epilogue: each accumulator row (one weight row) is multiplied by s[n] (int8 only), rounded to bf16 and staged
//     transposed ([token][weight row], 128B-swizzled) in shared memory; a TMA store writes D row-major and clips rows >= m,
//     columns >= n.
//   * When the output tiles leave SMs idle (decode), K is split: split j writes its fp32 partial product to the caller's
//     workspace and a second kernel sums the splits in order, scales (int8), rounds and stores D. The plan is a function of
//     (m, n, k) and the SM count only, so graph replays equal eager calls bit for bit.
//   * fsb_gemm_{w8a16,w4a16}_bias (GPT-2's Conv1D projections): the kEpi instantiations add bias[n] to the scaled sum and
//     optionally apply gelu_tanh_f (gemm_epilogue.cuh, the bf16 and FP8 GEMMs' device code) before the one rounding, in the
//     unsplit kernel's epilogue or, when K is split, in the reduce kernel after the splits are summed: once per element. The
//     plain instantiations (fsb_gemm_w8a16 / fsb_gemm_w4a16) carry none of that code.
#include "gemm_epilogue.cuh"
#include "host_common.h"
#include "ptx.cuh"

namespace fsb {

constexpr int W8_BM = 128;        // weight rows per tile (2 consumer warpgroups x 64)
constexpr int W8_BK = 128;        // k per stage: one 128-byte swizzle line of int8 per row, of int4 per row pair
constexpr int W8_THREADS = 384;
constexpr int W4_GROUP = 128;     // int4: k per scale group (= W8_BK: one group per stage)

// int8: a 128-byte line of the weight tile is one weight row; a thread's fragment rows are `row` and `row + 8`; the fp32
// per-row scale is applied after the sum.
struct FmtW8 {
  static constexpr int kRowsPerLine = 1;
  static constexpr int kPartner = 8;        // the thread's second weight row is row + kPartner
  static constexpr int kMaxStages = 8;
  static constexpr bool kRowScale = true;
};
// int4: a line is a row pair (2p, 2p + 1) and a thread's fragment rows are `row` (even) and `row + 1`; the group scales are
// applied to the fragments, so the sum is stored as it is. Half the bytes per stage: up to twice the stages keeps as many
// weight bytes in flight as int8.
struct FmtW4 {
  static constexpr int kRowsPerLine = 2;
  static constexpr int kPartner = 1;
  static constexpr int kMaxStages = 16;
  static constexpr bool kRowScale = false;
};

template <class F, int BT>
struct WqSmem {
  static constexpr int W_BYTES = W8_BM / F::kRowsPerLine * 128;  // quantised weight tile
  static constexpr int T_BYTES = BT * W8_BK * 2;               // two 64-wide bf16 token boxes
  static constexpr int STAGE_BYTES = W_BYTES + T_BYTES;
  static constexpr int EPI_BYTES = 2 * BT * 128;               // per consumer warpgroup: BT tokens x 64 bf16 weight rows
  static constexpr int BUDGET = kSmemOptIn - 1024 - 256;
  static constexpr int FIT = (BUDGET - EPI_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = FIT > F::kMaxStages ? F::kMaxStages : FIT;
  static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = EPI_OFFSET + EPI_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8 + 1024 /*align slack*/;
  static_assert(STAGES >= 3, "too few pipeline stages");
  static_assert(2 * STAGES * 8 <= 256, "barriers exceed their reserve");
  static_assert(TOTAL <= kSmemOptIn, "exceeds the 227 KB of shared memory a block can opt into on sm_90");
  static_assert(STAGE_BYTES % 1024 == 0 && (BT * 128) % 1024 == 0, "swizzled tiles must stay 1024-byte aligned");
};

struct WqParams {
  const void* scale;  // int8: fp32 [N]; int4: bf16 [N, K / 128]
  float* ws;          // split-K partials [splits, M, N] fp32, or nullptr
  int M, N, K;
  int tiles_t, tiles_n, splits, num_kb;
  const __nv_bfloat16* bias;   // [N]; read by the kEpi instantiations only (appended: the plain ones keep their offsets)
};

// The epilogue forms: what happens to the fp32 sum (scaled by s[n] for int8) before its one rounding to bf16
constexpr int WQ_PLAIN = 0;       // nothing (fsb_gemm_w8a16 / fsb_gemm_w4a16)
constexpr int WQ_BIAS = 1;        // + bias[n]
constexpr int WQ_BIAS_GELU = 2;   // gelu_tanh(. + bias[n]) (GPT-2's c_fc: gelu_new)

template <int kEpi>
__device__ __forceinline__ float wq_epilogue(float v, float b) {
  if constexpr (kEpi != WQ_PLAIN) {
    v = __fadd_rn(v, b);   // never contracted with the int8 scale multiply: the unsplit and split paths round alike
    if constexpr (kEpi == WQ_BIAS_GELU) v = gelu_tanh_f(v);
  }
  return v;
}

// Four int8 (bytes of x) -> two bf16x2 (bytes 0,1 -> lo; bytes 2,3 -> hi), exactly: x + 128 is placed in the mantissa of
// 2^23 (fp32 0x4B000000 | (x ^ 0x80)), 2^23 + 128 is subtracted, and the integer result, at most 8 significant bits, keeps its
// value in the upper half of the fp32 word (a bf16).
__device__ __forceinline__ void i8x4_to_bf16x4(uint32_t x, uint32_t& lo, uint32_t& hi) {
  x ^= 0x80808080u;
  const float f0 = __uint_as_float(__byte_perm(x, 0x4B000000u, 0x7540)) - 8388736.f;
  const float f1 = __uint_as_float(__byte_perm(x, 0x4B000000u, 0x7541)) - 8388736.f;
  const float f2 = __uint_as_float(__byte_perm(x, 0x4B000000u, 0x7542)) - 8388736.f;
  const float f3 = __uint_as_float(__byte_perm(x, 0x4B000000u, 0x7543)) - 8388736.f;
  lo = __byte_perm(__float_as_uint(f0), __float_as_uint(f1), 0x7632);
  hi = __byte_perm(__float_as_uint(f2), __float_as_uint(f3), 0x7632);
}

// Two int4 codes (bits 0-3 and 16-19 of x, each q + 8) -> the bf16x2 pair bf16(q * s), s2 holding s twice. 0x4300 | code is
// the bf16 128 + code; subtracting 136 gives q exactly, and one bf16 multiply rounds the exact product q * s once.
__device__ __forceinline__ uint32_t i4x2_to_bf16x2(uint32_t x, uint32_t s2) {
  const uint32_t v = (x & 0x000F000Fu) | 0x43004300u;
  uint32_t q, w;
  asm("fma.rn.bf16x2 %0, %1, %2, %3;" : "=r"(q) : "r"(v), "r"(0x3F803F80u), "r"(0xC308C308u));   // v * 1 - 136
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(w) : "r"(q), "r"(s2));
  return w;
}

template <class F, int BT, int kEpi>
__global__ void __launch_bounds__(W8_THREADS, 1)
gemm_wq_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmA,
               const __grid_constant__ CUtensorMap tmD, const WqParams p) {
  using S = WqSmem<F, BT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  TmaRing<S::STAGES> ring(reinterpret_cast<uint64_t*>(smem + S::BAR_OFFSET));

  // tile order: token tiles fastest, so the CTAs of a wave share weight tiles (prefill) through L2
  const int t_idx = blockIdx.x % p.tiles_t;
  const int rest = blockIdx.x / p.tiles_t;
  const int n_idx = rest % p.tiles_n;
  const int split = rest / p.tiles_n;
  const int kb_lo = int(int64_t(split) * p.num_kb / p.splits), kb_hi = int(int64_t(split + 1) * p.num_kb / p.splits);
  const int n0 = n_idx * W8_BM, t0 = t_idx * BT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmA);
    ring.init();
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    reg_dec<40>();
    if (threadIdx.x == 0) {
      for (int kb = kb_lo; kb < kb_hi; ++kb) {
        ring.acquire();
        uint8_t* sw = smem + ring.stage * S::STAGE_BYTES;
        uint8_t* st = sw + S::W_BYTES;
        const int k0 = kb * W8_BK;
        const bool second = k0 + 64 < p.K;   // the upper 64-wide token box holds real columns
        uint64_t* bar = ring.expect(S::W_BYTES + (second ? 2 : 1) * BT * 128);
        tma_load_2d(sw, &tmW, bar, k0, n0 / F::kRowsPerLine);   // int4: a byte line of q holds a row pair's k values
        tma_load_2d(st, &tmA, bar, k0, t0);
        if (second) tma_load_2d(st + BT * 128, &tmA, bar, k0 + 64, t0);
        ring.advance();
      }
    }
  } else {
    // ===================== consumers: warpgroup wg owns weight rows [64 wg, 64 wg + 64) of the tile =====================
    reg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int wl = warp & 3, g = lane >> 2, tq = lane & 3;
    const int row = wg * 64 + wl * 16 + F::kRowsPerLine * g;   // this thread's weight rows in the tile: row, row + kPartner
    const uint32_t smem_base = smem_u32(smem);
    const uint64_t dsc_t = make_smem_desc_sw128(smem_base + S::W_BYTES, 0, 1024);
    float acc[BT / 2];
#pragma unroll
    for (int i = 0; i < BT / 2; ++i) acc[i] = 0.f;
    // The consumer keeps its ring position in locals rather than in `ring`: with the position inside the closure of
    // run_stage, ptxas assigns registers differently and the kernel measured about 1 % slower on an H100 80GB HBM3 (700 W).
    uint64_t* const full_bar = ring.bar;
    uint64_t* const empty_bar = ring.empty_bar;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    // int4: the group scales of rows `row` and `row + 1` (bf16 bits), loaded one stage ahead. Rows at or beyond N read row
    // N - 2's scales: their sums are never stored.
    const uint16_t* s_row = nullptr;
    uint32_t s_next0 = 0, s_next1 = 0;
    if constexpr (!F::kRowScale) {
      s_row = static_cast<const uint16_t*>(p.scale) + int64_t(min(n0 + row, p.N - 2)) * p.num_kb;
      s_next0 = __ldg(s_row + kb_lo);
      s_next1 = __ldg(s_row + p.num_kb + kb_lo);
    }

    // One stage: convert this thread's fragments of the weight tile into `fr`, issue the stage's MMAs, then wait until the
    // PREVIOUS stage's MMAs have retired (its token tile and its fragment buffer, the other one, are then free).
    auto run_stage = [&](uint32_t (&fr)[8][4], int kb) {
      uint32_t sc0 = 0, sc1 = 0;
      if constexpr (!F::kRowScale) {
        sc0 = s_next0 * 0x10001u;
        sc1 = s_next1 * 0x10001u;
        const int nk = min(kb + 1, kb_hi - 1);
        s_next0 = __ldg(s_row + nk);
        s_next1 = __ldg(s_row + p.num_kb + nk);
      }
      mbar_wait(&full_bar[stage], phase);
      const int steps = min(8, (p.K - kb * W8_BK) >> 4);   // k16 steps inside K (K % 16 == 0)
      const uint32_t w0 = smem_base + stage * S::STAGE_BYTES;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        if (kk < steps) {
          if constexpr (F::kRowScale) {
            const uint32_t a = w0 + swz128(row, 16 * kk + 2 * tq);   // row + 8 is 1024 bytes on, same swizzle phase
            const uint32_t x = __byte_perm(lds_u16(a), lds_u16(a + 1024), 0x5410);
            const uint32_t y = __byte_perm(lds_u16(a + 8), lds_u16(a + 1024 + 8), 0x5410);
            uint32_t r0, r1, r2, r3;
            i8x4_to_bf16x4(x, r0, r1);
            i8x4_to_bf16x4(y, r2, r3);
            fr[kk][0] = r0; fr[kk][1] = r1; fr[kk][2] = r2; fr[kk][3] = r3;
          } else {
            // the row pair's line is row / 2 of the tile; a warp's 8 lines x 4 lanes hit 32 distinct banks
            const uint32_t x = lds_u32(w0 + swz128(row >> 1, 16 * kk + 4 * tq));
            fr[kk][0] = i4x2_to_bf16x2(x, sc0);         // (row, k..k+1)
            fr[kk][1] = i4x2_to_bf16x2(x >> 4, sc1);    // (row + 1, k..k+1)
            fr[kk][2] = i4x2_to_bf16x2(x >> 8, sc0);    // (row, k+8..k+9)
            fr[kk][3] = i4x2_to_bf16x2(x >> 12, sc1);   // (row + 1, k+8..k+9)
          }
        }
      }
      wgmma_fence();
      const uint64_t so = uint64_t(stage) * (S::STAGE_BYTES >> 4);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        if (kk < steps) {
          const uint64_t db = dsc_t + so + (uint64_t((kk >> 2) * BT * 128 + (kk & 3) * 32) >> 4);
          wgmma_rs_dim<BT, 0>(acc, fr[kk], db, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == S::STAGES) { stage = 0; phase ^= 1; }
    };
    uint32_t frA[8][4], frB[8][4];
    int kb = kb_lo;
    for (; kb + 1 < kb_hi; kb += 2) {
      run_stage(frA, kb);
      run_stage(frB, kb + 1);
    }
    if (kb < kb_hi) run_stage(frA, kb);
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

    // ---- epilogue: acc[4 j + 2 h + e] is (weight row `row + kPartner h`, token 8 j + 2 tq + e) of the tile
    const int nrow0 = n0 + row, nrow1 = nrow0 + F::kPartner;
    if (p.ws != nullptr) {
      // K-split: unscaled fp32 partial to ws[split, token, n]
      float* ws = p.ws + int64_t(split) * p.M * p.N;
#pragma unroll
      for (int j = 0; j < BT / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int tok = t0 + 8 * j + 2 * tq + e;
          if (tok >= p.M) continue;
          if (nrow0 < p.N) ws[int64_t(tok) * p.N + nrow0] = acc[4 * j + e];
          if (nrow1 < p.N) ws[int64_t(tok) * p.N + nrow1] = acc[4 * j + 2 + e];
        }
    } else {
      float s0 = 1.f, s1 = 1.f;
      if constexpr (F::kRowScale) {
        const float* scale = static_cast<const float*>(p.scale);
        s0 = nrow0 < p.N ? __ldg(scale + nrow0) : 0.f;
        s1 = nrow1 < p.N ? __ldg(scale + nrow1) : 0.f;
      }
      float b0 = 0.f, b1 = 0.f;
      if constexpr (kEpi != WQ_PLAIN) {
        b0 = nrow0 < p.N ? __bfloat162float(__ldg(p.bias + nrow0)) : 0.f;
        b1 = nrow1 < p.N ? __bfloat162float(__ldg(p.bias + nrow1)) : 0.f;
      }
      uint8_t* buf = smem + S::EPI_OFFSET + wg * (BT * 128);
      const int lr = wl * 16 + F::kRowsPerLine * g;   // weight row inside the warpgroup's 64 (the staging tile's column)
#pragma unroll
      for (int j = 0; j < BT / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int tok = 8 * j + 2 * tq + e;
          *reinterpret_cast<__nv_bfloat16*>(buf + swz128(tok, 2 * lr)) =
              __float2bfloat16_rn(wq_epilogue<kEpi>(acc[4 * j + e] * s0, b0));
          *reinterpret_cast<__nv_bfloat16*>(buf + swz128(tok, 2 * (lr + F::kPartner))) =
              __float2bfloat16_rn(wq_epilogue<kEpi>(acc[4 * j + 2 + e] * s1, b1));
        }
      fence_proxy_async();
      bar_sync(1 + wg, 128);
      if ((threadIdx.x & 127) == 0 && n0 + wg * 64 < p.N) {
        tma_store_2d(&tmD, buf, n0 + wg * 64, t0);
        tma_store_commit();
        tma_store_wait<0>();
      }
    }
  }
}

// D[m, n:n+8] = bf16(s[n:n+8] * sum over splits of ws[split, m, n:n+8]), splits summed in order; int4 (kRowScale false)
// stores the sum unscaled. kEpi: then the bias / GELU of wq_epilogue, as the unsplit kernel applies them (bias: the last
// parameter, read by those instantiations only).
template <bool kRowScale, int kEpi>
__global__ void wq_splitk_reduce_kernel(const float* __restrict__ ws, const float* __restrict__ scale, int splits, int64_t M,
                                        int64_t N, __nv_bfloat16* __restrict__ D, int64_t ldd,
                                        const __nv_bfloat16* __restrict__ bias) {
  const int64_t n8 = N / 8;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < M * n8; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t m = i / n8, n = (i - m * n8) * 8;
    float v[8];
    const float4* src = reinterpret_cast<const float4*>(ws + m * N + n);
    float4 a = src[0], b = src[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    for (int s = 1; s < splits; ++s) {
      const float4* q = reinterpret_cast<const float4*>(ws + (int64_t(s) * M + m) * N + n);
      a = q[0]; b = q[1];
      v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
    }
    if constexpr (kRowScale) {
      const float4 s0 = *reinterpret_cast<const float4*>(scale + n), s1 = *reinterpret_cast<const float4*>(scale + n + 4);
      v[0] *= s0.x; v[1] *= s0.y; v[2] *= s0.z; v[3] *= s0.w; v[4] *= s1.x; v[5] *= s1.y; v[6] *= s1.z; v[7] *= s1.w;
    }
    if constexpr (kEpi != WQ_PLAIN) {
      const uint4 bv = *reinterpret_cast<const uint4*>(bias + n);
      v[0] = wq_epilogue<kEpi>(v[0], bf16lo(bv.x)); v[1] = wq_epilogue<kEpi>(v[1], bf16hi(bv.x));
      v[2] = wq_epilogue<kEpi>(v[2], bf16lo(bv.y)); v[3] = wq_epilogue<kEpi>(v[3], bf16hi(bv.y));
      v[4] = wq_epilogue<kEpi>(v[4], bf16lo(bv.z)); v[5] = wq_epilogue<kEpi>(v[5], bf16hi(bv.z));
      v[6] = wq_epilogue<kEpi>(v[6], bf16lo(bv.w)); v[7] = wq_epilogue<kEpi>(v[7], bf16hi(bv.w));
    }
    *reinterpret_cast<uint4*>(D + m * ldd + n) = pack8(v);
  }
}

// One block per row: s = absmax / 127 (IEEE division), q = clamp(rint(w / s), -127, 127); a zero row gives s = 0, q = 0
__global__ void quantize_w8_kernel(const __nv_bfloat16* __restrict__ W, int64_t ldw, int64_t K, int8_t* __restrict__ q,
                                   float* __restrict__ s) {
  __shared__ float red[32];
  const __nv_bfloat16* w = W + int64_t(blockIdx.x) * ldw;
  float amax = 0.f;
  for (int64_t c = threadIdx.x; c < K; c += blockDim.x) amax = fmaxf(amax, fabsf(__bfloat162float(w[c])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (threadIdx.x == 0) red[0] = v;
  }
  __syncthreads();
  const float sc = __fdiv_rn(red[0], 127.0f);
  if (threadIdx.x == 0) s[blockIdx.x] = sc;
  int8_t* qr = q + int64_t(blockIdx.x) * K;
  for (int64_t c = threadIdx.x; c < K; c += blockDim.x) {
    float v = 0.f;
    if (sc != 0.f) v = fminf(fmaxf(rintf(__fdiv_rn(__bfloat162float(w[c]), sc)), -127.f), 127.f);
    qr[c] = static_cast<int8_t>(v);
  }
}

// One warp per (row pair 2p, 2p + 1; group of 128 k), 8 groups per block: per row s = bf16(absmax / 7) (IEEE division, then
// round to nearest even), q = clamp(rint(w / s), -7, 7) (0 where s == 0), packed as include/fsb200.h lays it out: in each
// 16-k block, byte 4t + 2b + h holds k = 8h + 2t + b, row 2p in the low nibble and row 2p + 1 in the high one, each q + 8.
__global__ void quantize_w4_kernel(const __nv_bfloat16* __restrict__ W, int64_t ldw, int64_t K, int groups,
                                   uint8_t* __restrict__ q, __nv_bfloat16* __restrict__ s) {
  __shared__ int8_t qs[8][2][W4_GROUP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = blockIdx.y * 8 + warp;
  if (grp >= groups) return;
  const int64_t pr = blockIdx.x;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const __nv_bfloat16* w = W + (2 * pr + e) * ldw + int64_t(grp) * W4_GROUP + 4 * lane;
    float v[4], amax = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      v[i] = __bfloat162float(w[i]);
      amax = fmaxf(amax, fabsf(v[i]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const __nv_bfloat16 sb = __float2bfloat16_rn(__fdiv_rn(amax, 7.0f));
    const float sc = __bfloat162float(sb);
    if (lane == 0) s[(2 * pr + e) * groups + grp] = sb;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float r = 0.f;
      if (sc != 0.f) r = fminf(fmaxf(rintf(__fdiv_rn(v[i], sc)), -7.f), 7.f);
      qs[warp][e][4 * lane + i] = static_cast<int8_t>(r);
    }
  }
  __syncwarp();
  // this lane writes bytes 4 lane .. 4 lane + 3 of the group: 16-k block lane / 4, t = lane % 4, byte i = 2b + h
  uint32_t word = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = 16 * (lane >> 2) + 8 * (i & 1) + 2 * (lane & 3) + (i >> 1);
    word |= uint32_t((qs[warp][0][c] + 8) | ((qs[warp][1][c] + 8) << 4)) << (8 * i);
  }
  reinterpret_cast<uint32_t*>(q + pr * K + int64_t(grp) * W4_GROUP)[lane] = word;
}

// Token-tile width and K-split count, from (m, n, k) and the SM count only. Tiles are 128 weight rows x BT tokens, BT the
// smallest of 8, 16, 32, 64, 128 that holds m (decode fits in one token tile). Too few tiles for the SMs (decode: n = 5120
// is 40 tiles) split K into equal runs of whole 128-deep blocks, the smallest count whose waves keep >= 90% of the SMs busy
// (else the best), each run at least 2 blocks deep. Both weight formats use the same plan.
struct W8Plan {
  int bt, splits;
};
static W8Plan w8_plan(int64_t M, int64_t N, int64_t K, int sms) {
  const int bt = M <= 8 ? 8 : M <= 16 ? 16 : M <= 32 ? 32 : M <= 64 ? 64 : 128;
  const int64_t tiles = ((N + W8_BM - 1) / W8_BM) * ((M + bt - 1) / bt);
  const int64_t num_kb = (K + W8_BK - 1) / W8_BK;
  if (tiles >= 2 * int64_t(sms)) return {bt, 1};
  int best = 1;
  double best_eff = 0.0;
  for (int s = 1; s <= 16 && (s == 1 || num_kb / s >= 2); ++s) {
    const int64_t units = tiles * s, waves = (units + sms - 1) / sms;
    const double eff = double(units) / double(waves * sms);
    if (eff > best_eff + 1e-9) { best = s; best_eff = eff; }
    if (eff >= 0.9) break;
  }
  return {bt, best};
}

static size_t wq_workspace_bytes(int64_t m, int64_t n, int64_t k) {
  if (m <= 0 || n <= 0 || k <= 0) return 0;
  const W8Plan plan = w8_plan(m, n, k, num_sms());
  return plan.splits > 1 ? size_t(plan.splits) * size_t(m) * size_t(n) * sizeof(float) : 0;
}

template <class F, int BT, int kEpi>
static int launch_wq(const CUtensorMap& tmW, const CUtensorMap& tmA, const CUtensorMap& tmD, const WqParams& p,
                     cudaStream_t stream, const char* what) {
  using S = WqSmem<F, BT>;
  if (int rc = ensure_smem<gemm_wq_kernel<F, BT, kEpi>>(S::TOTAL, what)) return rc;
  const int64_t grid = int64_t(p.tiles_t) * p.tiles_n * p.splits;
  gemm_wq_kernel<F, BT, kEpi><<<unsigned(grid), W8_THREADS, S::TOTAL, stream>>>(tmW, tmA, tmD, p);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

// The GEMM kernel for the plan's token-tile width, then (K split) the reduce kernel
template <class F, int kEpi>
static int run_wq(const CUtensorMap& tmW, const CUtensorMap& tmA, const CUtensorMap& tmD, const WqParams& p, int bt,
                  int64_t m, int64_t n, const void* s, void* d, int64_t ldd, cudaStream_t stream, const char* what) {
  int rc = FSB_ERR_INVALID;
  switch (bt) {
    case 8: rc = launch_wq<F, 8, kEpi>(tmW, tmA, tmD, p, stream, what); break;
    case 16: rc = launch_wq<F, 16, kEpi>(tmW, tmA, tmD, p, stream, what); break;
    case 32: rc = launch_wq<F, 32, kEpi>(tmW, tmA, tmD, p, stream, what); break;
    case 64: rc = launch_wq<F, 64, kEpi>(tmW, tmA, tmD, p, stream, what); break;
    default: rc = launch_wq<F, 128, kEpi>(tmW, tmA, tmD, p, stream, what); break;
  }
  if (rc || p.splits == 1) return rc;
  const int64_t work = m * (n / 8);
  const int blocks = int(work / 256 + 1 < 4 * num_sms() ? work / 256 + 1 : 4 * num_sms());
  wq_splitk_reduce_kernel<F::kRowScale, kEpi><<<blocks, 256, 0, stream>>>(
      p.ws, static_cast<const float*>(F::kRowScale ? s : nullptr), p.splits, m, n, static_cast<__nv_bfloat16*>(d), ldd,
      p.bias);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

// The checks and launch shared by fsb_gemm_{w8a16,w4a16}[_bias] (`what` names the entry in messages). The format's own
// k requirement is checked by the caller. bias == nullptr: the plain GEMM (epilogue ignored); otherwise `epilogue`, already
// checked to be FSB_EPI_NONE or FSB_EPI_GELU_TANH, selects the bias form.
template <class F>
static int gemm_wq(const char* what, int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const void* q,
                   const void* s, const void* bias, int epilogue, void* d, int64_t ldd, void* workspace,
                   size_t workspace_bytes, cudaStream_t stream) {
  FSB_REQUIRE(n % 8 == 0, "%s: n=%ld must be a multiple of 8", what, (long)n);
  FSB_REQUIRE(a && q && s && d, "%s: null operand", what);
  FSB_REQUIRE(aligned16(a) && aligned16(q) && aligned16(s) && aligned16(d), "%s: a, q, s and d must be 16-byte aligned",
              what);
  FSB_REQUIRE(lda >= k && lda % 8 == 0, "%s: lda=%ld must be >= k and a multiple of 8", what, (long)lda);
  FSB_REQUIRE(ldd >= n && ldd % 8 == 0, "%s: ldd=%ld must be >= n and a multiple of 8", what, (long)ldd);
  const W8Plan plan = w8_plan(m, n, k, num_sms());
  const size_t need = plan.splits > 1 ? size_t(plan.splits) * size_t(m) * size_t(n) * sizeof(float) : 0;
  FSB_REQUIRE(need == 0 || (workspace != nullptr && workspace_bytes >= need && aligned16(workspace)),
              "%s: this call splits K %d ways and needs a 16-byte aligned %zu-byte workspace "
              "(fsb_%s_workspace_bytes); got %zu",
              what, plan.splits, need, what, workspace_bytes);

  CUtensorMap tmW, tmA, tmD;
  {
    // int8: [n, k] bytes; int4: [n / 2, k] bytes, a line per row pair
    uint64_t dims[2] = {uint64_t(k), uint64_t(n / F::kRowsPerLine)};
    uint64_t strides[1] = {uint64_t(k)};
    uint32_t box[2] = {uint32_t(W8_BK), uint32_t(W8_BM / F::kRowsPerLine)};
    int rc = make_tmap_u8(&tmW, q, 2, dims, strides, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {uint64_t(k), uint64_t(m)};
    uint64_t strides[1] = {uint64_t(lda) * 2};
    uint32_t box[2] = {64, uint32_t(plan.bt)};
    int rc = make_tmap_bf16(&tmA, a, 2, dims, strides, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {uint64_t(n), uint64_t(m)};
    uint64_t strides[1] = {uint64_t(ldd) * 2};
    uint32_t box[2] = {64, uint32_t(plan.bt)};
    int rc = make_tmap_bf16(&tmD, d, 2, dims, strides, box);
    if (rc) return rc;
  }
  WqParams p;
  p.scale = s;
  p.ws = plan.splits > 1 ? static_cast<float*>(workspace) : nullptr;
  p.M = int(m); p.N = int(n); p.K = int(k);
  p.tiles_t = int((m + plan.bt - 1) / plan.bt);
  p.tiles_n = int((n + W8_BM - 1) / W8_BM);
  p.splits = plan.splits;
  p.num_kb = int((k + W8_BK - 1) / W8_BK);
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  if (bias == nullptr) return run_wq<F, WQ_PLAIN>(tmW, tmA, tmD, p, plan.bt, m, n, s, d, ldd, stream, what);
  if (epilogue == FSB_EPI_GELU_TANH) return run_wq<F, WQ_BIAS_GELU>(tmW, tmA, tmD, p, plan.bt, m, n, s, d, ldd, stream, what);
  return run_wq<F, WQ_BIAS>(tmW, tmA, tmD, p, plan.bt, m, n, s, d, ldd, stream, what);
}

// The checks of the _bias entries' extra operands
static int check_wq_bias(const char* what, const void* bias, int epilogue) {
  FSB_REQUIRE(bias != nullptr, "%s: bias must not be NULL (the entry without _bias is the bias-free GEMM)", what);
  FSB_REQUIRE(aligned16(bias), "%s: bias must be 16-byte aligned", what);
  FSB_REQUIRE(epilogue == FSB_EPI_NONE || epilogue == FSB_EPI_GELU_TANH,
              "%s: epilogue=%d unsupported (FSB_EPI_NONE or FSB_EPI_GELU_TANH)", what, epilogue);
  return FSB_OK;
}

}  // namespace fsb

using namespace fsb;

extern "C" int fsb_quantize_w8(const void* w, int64_t ldw, int64_t n, int64_t k, int8_t* q, float* s, fsb_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FSB_REQUIRE(n > 0 && k > 0, "quantize_w8: non-positive dims n=%ld k=%ld", (long)n, (long)k);
  FSB_REQUIRE(n < (int64_t(1) << 31), "quantize_w8: n=%ld too large", (long)n);
  FSB_REQUIRE(ldw >= k, "quantize_w8: ldw=%ld < k=%ld", (long)ldw, (long)k);
  FSB_REQUIRE(w && q && s, "quantize_w8: null pointer");
  FSB_REQUIRE((reinterpret_cast<uintptr_t>(w) & 1) == 0 && (reinterpret_cast<uintptr_t>(s) & 3) == 0,
              "quantize_w8: misaligned w or s");
  quantize_w8_kernel<<<unsigned(n), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(w), ldw, k, q, s);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

extern "C" size_t fsb_gemm_w8a16_workspace_bytes(int64_t m, int64_t n, int64_t k) { return wq_workspace_bytes(m, n, k); }

extern "C" int fsb_gemm_w8a16(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const int8_t* q,
                              const float* s, void* d, int64_t ldd, void* workspace, size_t workspace_bytes,
                              fsb_stream_t stream_) {
  FSB_REQUIRE(m > 0 && n > 0 && k > 0, "gemm_w8a16: non-positive dims m=%ld n=%ld k=%ld", (long)m, (long)n, (long)k);
  FSB_REQUIRE(m < (1 << 30) && n < (1 << 30) && k < (1 << 30), "gemm_w8a16: dims too large");
  FSB_REQUIRE(k % 16 == 0, "gemm_w8a16: k=%ld must be a multiple of 16", (long)k);
  return gemm_wq<FmtW8>("gemm_w8a16", m, n, k, a, lda, q, s, nullptr, FSB_EPI_NONE, d, ldd, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream_));
}

extern "C" int fsb_gemm_w8a16_bias(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const int8_t* q,
                                   const float* s, const void* bias, int epilogue, void* d, int64_t ldd, void* workspace,
                                   size_t workspace_bytes, fsb_stream_t stream_) {
  FSB_REQUIRE(m > 0 && n > 0 && k > 0, "gemm_w8a16_bias: non-positive dims m=%ld n=%ld k=%ld", (long)m, (long)n, (long)k);
  FSB_REQUIRE(m < (1 << 30) && n < (1 << 30) && k < (1 << 30), "gemm_w8a16_bias: dims too large");
  FSB_REQUIRE(k % 16 == 0, "gemm_w8a16_bias: k=%ld must be a multiple of 16", (long)k);
  if (int rc = check_wq_bias("gemm_w8a16_bias", bias, epilogue)) return rc;
  // the plan and its workspace are fsb_gemm_w8a16's: named after it in the workspace message
  return gemm_wq<FmtW8>("gemm_w8a16", m, n, k, a, lda, q, s, bias, epilogue, d, ldd, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream_));
}

extern "C" int fsb_quantize_w4(const void* w, int64_t ldw, int64_t n, int64_t k, uint8_t* q, void* s,
                               fsb_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FSB_REQUIRE(n > 0 && k > 0, "quantize_w4: non-positive dims n=%ld k=%ld", (long)n, (long)k);
  FSB_REQUIRE(n < (int64_t(1) << 31) && k < (int64_t(1) << 30), "quantize_w4: n=%ld or k=%ld too large", (long)n, (long)k);
  FSB_REQUIRE(k % W4_GROUP == 0, "quantize_w4: k=%ld must be a multiple of %d (the scale group)", (long)k, W4_GROUP);
  FSB_REQUIRE(n % 8 == 0, "quantize_w4: n=%ld must be a multiple of 8", (long)n);
  FSB_REQUIRE(ldw >= k, "quantize_w4: ldw=%ld < k=%ld", (long)ldw, (long)k);
  FSB_REQUIRE(w && q && s, "quantize_w4: null pointer");
  FSB_REQUIRE((reinterpret_cast<uintptr_t>(w) & 1) == 0 && (reinterpret_cast<uintptr_t>(q) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(s) & 1) == 0,
              "quantize_w4: misaligned w, q or s");
  const int groups = int(k / W4_GROUP);
  const dim3 grid(unsigned(n / 2), unsigned((groups + 7) / 8));
  quantize_w4_kernel<<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(w), ldw, k, groups, q,
                                               static_cast<__nv_bfloat16*>(s));
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

extern "C" size_t fsb_gemm_w4a16_workspace_bytes(int64_t m, int64_t n, int64_t k) { return wq_workspace_bytes(m, n, k); }

extern "C" int fsb_gemm_w4a16(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const uint8_t* q,
                              const void* s, void* d, int64_t ldd, void* workspace, size_t workspace_bytes,
                              fsb_stream_t stream_) {
  FSB_REQUIRE(m > 0 && n > 0 && k > 0, "gemm_w4a16: non-positive dims m=%ld n=%ld k=%ld", (long)m, (long)n, (long)k);
  FSB_REQUIRE(m < (1 << 30) && n < (1 << 30) && k < (1 << 30), "gemm_w4a16: dims too large");
  FSB_REQUIRE(k % W4_GROUP == 0, "gemm_w4a16: k=%ld must be a multiple of %d (the scale group)", (long)k, W4_GROUP);
  return gemm_wq<FmtW4>("gemm_w4a16", m, n, k, a, lda, q, s, nullptr, FSB_EPI_NONE, d, ldd, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream_));
}

extern "C" int fsb_gemm_w4a16_bias(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const uint8_t* q,
                                   const void* s, const void* bias, int epilogue, void* d, int64_t ldd, void* workspace,
                                   size_t workspace_bytes, fsb_stream_t stream_) {
  FSB_REQUIRE(m > 0 && n > 0 && k > 0, "gemm_w4a16_bias: non-positive dims m=%ld n=%ld k=%ld", (long)m, (long)n, (long)k);
  FSB_REQUIRE(m < (1 << 30) && n < (1 << 30) && k < (1 << 30), "gemm_w4a16_bias: dims too large");
  FSB_REQUIRE(k % W4_GROUP == 0, "gemm_w4a16_bias: k=%ld must be a multiple of %d (the scale group)", (long)k, W4_GROUP);
  if (int rc = check_wq_bias("gemm_w4a16_bias", bias, epilogue)) return rc;
  return gemm_wq<FmtW4>("gemm_w4a16", m, n, k, a, lda, q, s, bias, epilogue, d, ldd, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream_));
}
