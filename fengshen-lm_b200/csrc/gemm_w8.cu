// fsb200 — int8 weight-only GEMM (W8A16) and its quantiser for sm_90a: the inference layers behind `load_in_8bit=True`
// (fengshen/examples/ziya_inference/hf_quantizatin_inference.py:20-22, which hands the Linear layers to bitsandbytes'
// Linear8bitLt). Weights are stored as int8 q[n, k] with one fp32 scale per output channel, s[n] = absmax(W[n, :]) / 127;
// the GEMM computes D[m, n] = bf16(s[n] * sum_k A[m, k] q[n, k]) with fp32 accumulation.
//
// The operands are swapped against gemm.cu: decode has 1-32 token rows, far below the 64-row minimum of a wgmma A operand, so
// the WEIGHT tile is the A operand and the token tile the B operand (n = 8..128 tokens per tile).
//   * Roles (384 threads = 3 warpgroups): warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, each owning
//     64 of the tile's 128 weight rows.
//   * Per stage the producer loads a 128-row x 128-byte int8 weight tile and two 64-wide bf16 token boxes, all 128B-swizzled;
//     TMA zero-fills token rows at or beyond m and weight rows at or beyond n.
//   * Each consumer thread reads its fragment of the int8 tile (2-byte pieces: (row, k..k+1) as the register-A layout places
//     them), converts it to bf16 in registers (exact: every int8 is a bf16) and issues wgmma in the register-A form against
//     the token tile in shared memory. Two fragment buffers let one stage's conversion overlap the previous stage's MMAs.
//   * Epilogue: each accumulator row (one weight row) is multiplied by s[n], rounded to bf16 and staged transposed
//     ([token][weight row], 128B-swizzled) in shared memory; a TMA store writes D row-major and clips rows >= m, columns >= n.
//   * When the output tiles leave SMs idle (decode), K is split: split j writes its fp32 partial product to the caller's
//     workspace and a second kernel sums the splits in order, scales, rounds and stores D. The plan is a function of (m, n, k)
//     and the SM count only, so graph replays equal eager calls bit for bit.
#include "host_common.h"
#include "ptx.cuh"

namespace fsb {

constexpr int W8_BM = 128;        // weight rows per tile (2 consumer warpgroups x 64)
constexpr int W8_BK = 128;        // k per stage: one 128-byte swizzle row of int8
constexpr int W8_THREADS = 384;

template <int BT>
struct W8Smem {
  static constexpr int W_BYTES = W8_BM * W8_BK;                // int8 weight tile
  static constexpr int T_BYTES = BT * W8_BK * 2;               // two 64-wide bf16 token boxes
  static constexpr int STAGE_BYTES = W_BYTES + T_BYTES;
  static constexpr int EPI_BYTES = 2 * BT * 128;               // per consumer warpgroup: BT tokens x 64 bf16 weight rows
  static constexpr int BUDGET = kSmemOptIn - 1024 - 256;
  static constexpr int FIT = (BUDGET - EPI_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = FIT > 8 ? 8 : FIT;
  static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = EPI_OFFSET + EPI_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8 + 1024 /*align slack*/;
  static_assert(STAGES >= 3, "too few pipeline stages");
  static_assert(TOTAL <= kSmemOptIn, "exceeds the 227 KB of shared memory a block can opt into on sm_90");
  static_assert(STAGE_BYTES % 1024 == 0 && (BT * 128) % 1024 == 0, "swizzled tiles must stay 1024-byte aligned");
};

struct W8Params {
  const float* scale;
  float* ws;          // split-K partials [splits, M, N] fp32, or nullptr
  int M, N, K;
  int tiles_t, tiles_n, splits, num_kb;
};

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

template <int BT>
__global__ void __launch_bounds__(W8_THREADS, 1)
gemm_w8a16_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmA,
                  const __grid_constant__ CUtensorMap tmD, const W8Params p) {
  using S = W8Smem<BT>;
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
        tma_load_2d(sw, &tmW, bar, k0, n0);
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
    const int row = wg * 64 + wl * 16 + g;           // this thread's weight rows in the tile: row and row + 8
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

    // One stage: convert this thread's fragments of the int8 tile into `fr`, issue the stage's MMAs, then wait until the
    // PREVIOUS stage's MMAs have retired (its token tile and its fragment buffer, the other one, are then free).
    auto run_stage = [&](uint32_t (&fr)[8][4], int kb) {
      mbar_wait(&full_bar[stage], phase);
      const int steps = min(8, (p.K - kb * W8_BK) >> 4);   // k16 steps inside K (K % 16 == 0)
      const uint32_t w0 = smem_base + stage * S::STAGE_BYTES;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        if (kk < steps) {
          const uint32_t a = w0 + swz128(row, 16 * kk + 2 * tq);   // row + 8 is 1024 bytes on, same swizzle phase
          const uint32_t x = __byte_perm(lds_u16(a), lds_u16(a + 1024), 0x5410);
          const uint32_t y = __byte_perm(lds_u16(a + 8), lds_u16(a + 1024 + 8), 0x5410);
          uint32_t r0, r1, r2, r3;
          i8x4_to_bf16x4(x, r0, r1);
          i8x4_to_bf16x4(y, r2, r3);
          fr[kk][0] = r0; fr[kk][1] = r1; fr[kk][2] = r2; fr[kk][3] = r3;
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

    // ---- epilogue: acc[4 j + 2 h + e] is (weight row `row + 8 h`, token 8 j + 2 tq + e) of the tile
    const int nrow0 = n0 + row, nrow1 = nrow0 + 8;
    if (p.ws != nullptr) {
      // K-split: unscaled fp32 partial to ws[split, token, n]; a warp's 8 consecutive rows are 32 contiguous bytes per token
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
      const float s0 = nrow0 < p.N ? __ldg(p.scale + nrow0) : 0.f;
      const float s1 = nrow1 < p.N ? __ldg(p.scale + nrow1) : 0.f;
      uint8_t* buf = smem + S::EPI_OFFSET + wg * (BT * 128);
      const int lr = wl * 16 + g;   // weight row inside the warpgroup's 64 (the staging tile's column)
#pragma unroll
      for (int j = 0; j < BT / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int tok = 8 * j + 2 * tq + e;
          *reinterpret_cast<__nv_bfloat16*>(buf + swz128(tok, 2 * lr)) = __float2bfloat16_rn(acc[4 * j + e] * s0);
          *reinterpret_cast<__nv_bfloat16*>(buf + swz128(tok, 2 * (lr + 8))) = __float2bfloat16_rn(acc[4 * j + 2 + e] * s1);
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

// D[m, n:n+8] = bf16(s[n:n+8] * sum over splits of ws[split, m, n:n+8]), splits summed in order
__global__ void w8_splitk_reduce_kernel(const float* __restrict__ ws, const float* __restrict__ scale, int splits, int64_t M,
                                        int64_t N, __nv_bfloat16* __restrict__ D, int64_t ldd) {
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
    const float4 s0 = *reinterpret_cast<const float4*>(scale + n), s1 = *reinterpret_cast<const float4*>(scale + n + 4);
    v[0] *= s0.x; v[1] *= s0.y; v[2] *= s0.z; v[3] *= s0.w; v[4] *= s1.x; v[5] *= s1.y; v[6] *= s1.z; v[7] *= s1.w;
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

// Token-tile width and K-split count, from (m, n, k) and the SM count only. Tiles are 128 weight rows x BT tokens, BT the
// smallest of 8, 16, 32, 64, 128 that holds m (decode fits in one token tile). Too few tiles for the SMs (decode: n = 5120
// is 40 tiles) split K into equal runs of whole 128-deep blocks, the smallest count whose waves keep >= 90% of the SMs busy
// (else the best), each run at least 2 blocks deep.
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

template <int BT>
static int launch_w8(const CUtensorMap& tmW, const CUtensorMap& tmA, const CUtensorMap& tmD, const W8Params& p,
                     cudaStream_t stream) {
  using S = W8Smem<BT>;
  if (int rc = ensure_smem<gemm_w8a16_kernel<BT>>(S::TOTAL, "gemm_w8a16")) return rc;
  const int64_t grid = int64_t(p.tiles_t) * p.tiles_n * p.splits;
  gemm_w8a16_kernel<BT><<<unsigned(grid), W8_THREADS, S::TOTAL, stream>>>(tmW, tmA, tmD, p);
  FSB_CUDA_LAUNCH_CHECK();
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

extern "C" size_t fsb_gemm_w8a16_workspace_bytes(int64_t m, int64_t n, int64_t k) {
  if (m <= 0 || n <= 0 || k <= 0) return 0;
  const W8Plan plan = w8_plan(m, n, k, num_sms());
  return plan.splits > 1 ? size_t(plan.splits) * size_t(m) * size_t(n) * sizeof(float) : 0;
}

extern "C" int fsb_gemm_w8a16(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const int8_t* q,
                              const float* s, void* d, int64_t ldd, void* workspace, size_t workspace_bytes,
                              fsb_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FSB_REQUIRE(m > 0 && n > 0 && k > 0, "gemm_w8a16: non-positive dims m=%ld n=%ld k=%ld", (long)m, (long)n, (long)k);
  FSB_REQUIRE(m < (1 << 30) && n < (1 << 30) && k < (1 << 30), "gemm_w8a16: dims too large");
  FSB_REQUIRE(k % 16 == 0, "gemm_w8a16: k=%ld must be a multiple of 16", (long)k);
  FSB_REQUIRE(n % 8 == 0, "gemm_w8a16: n=%ld must be a multiple of 8", (long)n);
  FSB_REQUIRE(a && q && s && d, "gemm_w8a16: null operand");
  FSB_REQUIRE(aligned16(a) && aligned16(q) && aligned16(s) && aligned16(d),
              "gemm_w8a16: a, q, s and d must be 16-byte aligned");
  FSB_REQUIRE(lda >= k && lda % 8 == 0, "gemm_w8a16: lda=%ld must be >= k and a multiple of 8", (long)lda);
  FSB_REQUIRE(ldd >= n && ldd % 8 == 0, "gemm_w8a16: ldd=%ld must be >= n and a multiple of 8", (long)ldd);
  const W8Plan plan = w8_plan(m, n, k, num_sms());
  const size_t need = plan.splits > 1 ? size_t(plan.splits) * size_t(m) * size_t(n) * sizeof(float) : 0;
  FSB_REQUIRE(need == 0 || (workspace != nullptr && workspace_bytes >= need && aligned16(workspace)),
              "gemm_w8a16: this call splits K %d ways and needs a 16-byte aligned %zu-byte workspace "
              "(fsb_gemm_w8a16_workspace_bytes); got %zu",
              plan.splits, need, workspace_bytes);

  CUtensorMap tmW, tmA, tmD;
  {
    uint64_t dims[2] = {uint64_t(k), uint64_t(n)};
    uint64_t strides[1] = {uint64_t(k)};
    uint32_t box[2] = {uint32_t(W8_BK), uint32_t(W8_BM)};
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
  W8Params p;
  p.scale = s;
  p.ws = plan.splits > 1 ? static_cast<float*>(workspace) : nullptr;
  p.M = int(m); p.N = int(n); p.K = int(k);
  p.tiles_t = int((m + plan.bt - 1) / plan.bt);
  p.tiles_n = int((n + W8_BM - 1) / W8_BM);
  p.splits = plan.splits;
  p.num_kb = int((k + W8_BK - 1) / W8_BK);
  int rc = FSB_ERR_INVALID;
  switch (plan.bt) {
    case 8: rc = launch_w8<8>(tmW, tmA, tmD, p, stream); break;
    case 16: rc = launch_w8<16>(tmW, tmA, tmD, p, stream); break;
    case 32: rc = launch_w8<32>(tmW, tmA, tmD, p, stream); break;
    case 64: rc = launch_w8<64>(tmW, tmA, tmD, p, stream); break;
    default: rc = launch_w8<128>(tmW, tmA, tmD, p, stream); break;
  }
  if (rc || plan.splits == 1) return rc;
  const int64_t work = m * (n / 8);
  const int blocks = int(work / 256 + 1 < 4 * num_sms() ? work / 256 + 1 : 4 * num_sms());
  w8_splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(p.ws, s, plan.splits, m, n, static_cast<__nv_bfloat16*>(d), ldd);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
