// fsb200 — persistent, warp-specialised bf16 GEMM for sm_90a: TMA -> 128B-swizzled smem -> wgmma (fp32 accumulators in
// registers) -> fused epilogue -> HBM. Replaces the cuBLAS calls behind F.linear on the reference hot path
// (fengshen/models/megatron/mpu/layers.py:347-360, :451-470; layers/transformer.py:136-172) and their autograd
// transposes. One kernel, three operand layouts:
//   NT  D = A[M,K] B[N,K]^T   both operands K-major          (forward)
//   NN  D = A[M,K] B[K,N]     B is MN-major in shared memory  (dgrad)
//   TN  D = A[K,M]^T B[K,N]   A and B MN-major                (wgrad)
// MN-major tiles are fetched as 64(mn) x 64(k) TMA boxes; the wgmma descriptor's leading-byte-offset walks the boxes and
// the instruction's transpose bit reads them as MN-major.
//
// Roles (384 threads = 3 warpgroups): warpgroup 0 = TMA producer (one thread issues; setmaxnreg gives its registers to the
// others), warpgroups 1-2 = consumers: each owns 64 rows of the 128 x BN tile, issues m64nBNk16 wgmmas on the shared stage
// and runs the epilogue (bias / activation / pre-activation copy / bf16 or fp32 store, optionally accumulating) straight from
// its accumulator registers. The producer runs up to STAGES k-blocks ahead, across tile boundaries, so the next tile's
// operands stream in during the epilogue. Grid = min(#tiles, #SMs); static round-robin tile order, grouped for L2.
#include <stdlib.h>

#include "host_common.h"
#include "ptx.cuh"

namespace fsb {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 384;

struct GemmParams {
  void* D;
  void* aux;
  const void* bias;
  int64_t ldd, ldaux, stride_d, stride_aux;
  int M, N, K, batch;
  int d_f32;       // D dtype: 0 bf16, 1 fp32
  int bias_f32;    // bias dtype
  int epilogue;    // fsb_gemm_epilogue
  int accumulate;  // D += result
  int tiles_m, tiles_n;
  int group_m;     // m-tiles per rasterisation group (see fsb_gemm_bf16)
  int l2_hints;    // bit 0: A panels evict-last, bit 1: B panels evict-first (FSB_GEMM_L2HINT)
};

template <int BN>
struct GemmSmem {
  static constexpr int STAGES = BN == 256 ? 4 : 6;
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  // full[STAGES], empty[STAGES]
  static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8 + 1024 /*align slack*/;
  static_assert(TOTAL <= 232448, "exceeds the 227 KB of shared memory a block can opt into on sm_90");
};

// 0.5 x (1 + tanh(u)) == x * sigmoid(2u) == x / (1 + 2^(-2 u log2 e)): two MUFU ops instead of tanhf's ~25 instructions
// (relative error ~1e-6, far below the bf16 rounding of the stored activation)
__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float k1 = 0.044715f, c = -2.f * 0.7978845608028654f * 1.4426950408889634f;
  const float t = ex2_approx(c * x * fmaf(k1, x * x, 1.f));
  return __fdividef(x, 1.f + t);
}
// 0.5 x (1 + erf(x / sqrt 2)) with erfc from Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, far below the bf16 rounding of the
// stored activation): erfc(z) ~= t (a1 + t (a2 + t (a3 + t (a4 + t a5)))) exp(-z^2), t = 1 / (1 + 0.3275911 z), z = |x| / sqrt 2.
// Written on erfc so that the negative branch (1 + erf = erfc(|z|)) has no cancellation. ~12 instructions instead of erff's ~40.
__device__ __forceinline__ float gelu_erf_f(float x) {
  const float z = fabsf(x) * 0.7071067811865476f;
  const float t = __fdividef(1.f, fmaf(0.3275911f, z, 1.f));
  float pl = fmaf(t, 1.061405429f, -1.453152027f);
  pl = fmaf(t, pl, 1.421413741f);
  pl = fmaf(t, pl, -0.284496736f);
  pl = fmaf(t, pl, 0.254829592f);
  const float erfc_z = pl * t * ex2_approx(-1.4426950408889634f * z * z);
  const float hx = 0.5f * x;
  return x >= 0.f ? fmaf(-hx, erfc_z, x) : hx * erfc_z;
}

__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int group_m, int& b, int& m_idx, int& n_idx) {
  const int per = tiles_m * tiles_n;
  b = t / per;
  int r = t - b * per;
  const int group_span = group_m * tiles_n;
  const int g = r / group_span;
  const int first_m = g * group_m;
  const int gsize = min(tiles_m - first_m, group_m);
  const int in_g = r - g * group_span;
  m_idx = first_m + in_g % gsize;
  n_idx = in_g / gsize;
}

template <int kLayout, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  constexpr bool A_MN = (kLayout == FSB_GEMM_TN);
  constexpr bool B_MN = (kLayout != FSB_GEMM_NT);
  using S = GemmSmem<BN>;
  constexpr int STAGES = S::STAGES;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.tiles_m * p.tiles_n * p.batch;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    reg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      // L2 policy (FSB_GEMM_L2HINT): tiles are walked m-fastest inside a group of m-tiles, so a group's A panels are read
      // again for every n-tile of the sweep (evict-last) while a B panel is used by the CTAs of one wave (evict-first).
      const uint64_t pol_a = (p.l2_hints & 1) ? kL2EvictLast : kL2EvictNormal, pol_b = (p.l2_hints & 2) ? kL2EvictFirst : kL2EvictNormal;
      const bool hints = (p.l2_hints & 3) != 0;
      auto load = [&](uint8_t* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2, uint64_t policy) {
        if (hints) tma_load_3d_hint(dst, tm, bar, c0, c1, c2, policy);
        else tma_load_3d(dst, tm, bar, c0, c1, c2);
      };
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int b, m_idx, n_idx;
        tile_coords(t, p.tiles_m, p.tiles_n, p.group_m, b, m_idx, n_idx);
        const int m0 = m_idx * GEMM_BM, n0 = n_idx * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * S::STAGE_BYTES;
          uint8_t* sb = sa + S::A_BYTES;
          mbar_expect_tx(&full_bar[stage], S::STAGE_BYTES);
          const int k0 = kb * GEMM_BK;
          if constexpr (!A_MN) {
            load(sa, &tmA, &full_bar[stage], k0, m0, b, pol_a);
          } else {
#pragma unroll
            for (int c = 0; c < GEMM_BM / 64; ++c)
              load(sa + c * (GEMM_BK * 128), &tmA, &full_bar[stage], m0 + c * 64, k0, b, pol_a);
          }
          if constexpr (!B_MN) {
            load(sb, &tmB, &full_bar[stage], k0, n0, b, pol_b);
          } else {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c)
              load(sb + c * (GEMM_BK * 128), &tmB, &full_bar[stage], n0 + c * 64, k0, b, pol_b);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====================
    reg_inc<232>();  // 256 * 232 + 128 * 40 = 64512
    const int wg = (threadIdx.x >> 7) - 1;
    const int wl = warp & 3;
    // A: K-major -> the warpgroup's 64 rows start 64 * 128 B into the stage; MN-major -> its own 64-wide m chunk
    const uint64_t dsc_a = A_MN ? make_smem_desc_sw128(smem_u32(smem) + wg * (GEMM_BK * 128), GEMM_BK * 128, 1024)
                                : make_smem_desc_sw128(smem_u32(smem) + wg * (64 * 128), 0, 1024);
    const uint64_t dsc_b = B_MN ? make_smem_desc_sw128(smem_u32(smem) + S::A_BYTES, GEMM_BK * 128, 1024)
                                : make_smem_desc_sw128(smem_u32(smem) + S::A_BYTES, 0, 1024);
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int b, m_idx, n_idx;
      tile_coords(t, p.tiles_m, p.tiles_n, p.group_m, b, m_idx, n_idx);
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t so = uint64_t(stage) * (S::STAGE_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) {
          const uint64_t da = dsc_a + so + ((A_MN ? k * 2048 : k * 32) >> 4), db = dsc_b + so + ((B_MN ? k * 2048 : k * 32) >> 4);
          if constexpr (BN == 256) wgmma_ss_n256<A_MN, B_MN>(acc, da, db, (kb | k) != 0 ? 1u : 0u);
          else wgmma_ss_n128<A_MN, B_MN>(acc, da, db, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage can be refilled
        if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      // ---- epilogue from registers: accumulator j covers columns 8 (j / 4) + 2 (lane % 4) + (j & 1), rows r and r + 8
      const int row0 = m_idx * GEMM_BM + wg * 64 + wl * 16 + (lane >> 2);
      const int colq = n_idx * BN + 2 * (lane & 3);
      const int64_t d_off = int64_t(b) * p.stride_d, aux_off = int64_t(b) * p.stride_aux;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = colq + 8 * j;
        if (col >= p.N) continue;
        const bool two = col + 1 < p.N;
        float bv0 = 0.f, bv1 = 0.f;
        if (p.bias != nullptr) {
          if (p.bias_f32) {
            bv0 = __ldg(reinterpret_cast<const float*>(p.bias) + col);
            if (two) bv1 = __ldg(reinterpret_cast<const float*>(p.bias) + col + 1);
          } else {
            bv0 = __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16*>(p.bias) + col));
            if (two) bv1 = __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16*>(p.bias) + col + 1));
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          if (row >= p.M) continue;
          float v0 = acc[4 * j + 2 * h] + bv0, v1 = acc[4 * j + 2 * h + 1] + bv1;
          if (p.aux != nullptr) {   // pre-activation copy (bf16)
            __nv_bfloat16* ap = reinterpret_cast<__nv_bfloat16*>(p.aux) + aux_off + int64_t(row) * p.ldaux + col;
            if (two) *reinterpret_cast<uint32_t*>(ap) = pack_bf16x2(v0, v1);
            else *ap = __float2bfloat16(v0);
          }
          if (p.epilogue == FSB_EPI_GELU_TANH) { v0 = gelu_tanh_f(v0); v1 = gelu_tanh_f(v1); }
          else if (p.epilogue == FSB_EPI_GELU_ERF) { v0 = gelu_erf_f(v0); v1 = gelu_erf_f(v1); }
          if (p.d_f32) {
            float* dp = reinterpret_cast<float*>(p.D) + d_off + int64_t(row) * p.ldd + col;
            if (two) {
              float2 q = make_float2(v0, v1);
              if (p.accumulate) { const float2 o = *reinterpret_cast<const float2*>(dp); q.x += o.x; q.y += o.y; }
              *reinterpret_cast<float2*>(dp) = q;
            } else {
              *dp = p.accumulate ? *dp + v0 : v0;
            }
          } else {
            __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(p.D) + d_off + int64_t(row) * p.ldd + col;
            if (two) {
              if (p.accumulate) {
                const uint32_t o = *reinterpret_cast<const uint32_t*>(dp);
                v0 += bf16lo(o); v1 += bf16hi(o);
              }
              *reinterpret_cast<uint32_t*>(dp) = pack_bf16x2(v0, v1);
            } else {
              *dp = __float2bfloat16(p.accumulate ? __bfloat162float(*dp) + v0 : v0);
            }
          }
        }
      }
    }
  }
}

// SMs left to concurrently running communication kernels (fsb_set_reserved_sms): a persistent GEMM CTA fills an SM
// (all of its registers), so a collective that overlaps backward would otherwise push GEMM CTAs into a second wave.
static int g_reserved_sms = 0;
static inline int gemm_sms() {
  const int n = num_sms() - g_reserved_sms;
  return n < 1 ? 1 : n;
}

template <int kLayout, int BN>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t stream) {
  using S = GemmSmem<BN>;
  static bool configured = false;
  auto kern = gemm_bf16_kernel<kLayout, BN>;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL);
    if (e != cudaSuccess) {
      set_error("gemm: cudaFuncSetAttribute(%d B smem) failed: %s", S::TOTAL, cudaGetErrorString(e));
      return FSB_ERR_CUDA;
    }
    configured = true;
  }
  const int num_tiles = p.tiles_m * p.tiles_n * p.batch;
  const int grid = num_tiles < gemm_sms() ? num_tiles : gemm_sms();
  kern<<<grid, GEMM_THREADS, S::TOTAL, stream>>>(tmA, tmB, p);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

// D (bf16 / fp32, optionally accumulated into) = sum over the K-splits of the fp32 partial products, in a fixed order
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, int splits, int64_t M, int64_t N, void* D, int64_t ldd,
                                     int d_f32, int accumulate) {
  const int64_t n4 = N / 4;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < M * n4; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t m = i / n4, n = (i - m * n4) * 4;
    float4 acc = *reinterpret_cast<const float4*>(ws + m * N + n);
    for (int s = 1; s < splits; ++s) {
      const float4 v = *reinterpret_cast<const float4*>(ws + (int64_t(s) * M + m) * N + n);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (d_f32) {
      float4* dp = reinterpret_cast<float4*>(reinterpret_cast<float*>(D) + m * ldd + n);
      if (accumulate) { const float4 o = *dp; acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w; }
      *dp = acc;
    } else {
      uint2* dp = reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(D) + m * ldd + n);
      if (accumulate) {
        const uint2 o = *dp;
        acc.x += bf16lo(o.x); acc.y += bf16hi(o.x); acc.z += bf16lo(o.y); acc.w += bf16hi(o.y);
      }
      *dp = make_uint2(pack_bf16x2(acc.x, acc.y), pack_bf16x2(acc.z, acc.w));
    }
  }
}

static int gemm_impl(int layout, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                     int64_t ldb, void* D, int64_t ldd, int d_dtype, const void* bias, int bias_dtype,
                     int epilogue, int accumulate, void* aux, int64_t ldaux, int64_t batch, int64_t stride_a,
                     int64_t stride_b, int64_t stride_d, int64_t stride_aux, cudaStream_t stream, bool force_wide = false);

}  // namespace fsb

using namespace fsb;

extern "C" int fsb_set_reserved_sms(int n) {
  FSB_REQUIRE(n >= 0 && n <= 64, "set_reserved_sms: %d out of range [0, 64]", n);
  fsb::g_reserved_sms = n;
  return FSB_OK;
}

// Split-K plan for weight-gradient GEMMs whose output has too few tiles to occupy the SMs (e.g. 768 x 768 x 32768: 18
// tiles): `splits` K-chunks run as a batched GEMM into an fp32 scratch and are summed in a fixed order (deterministic).
// Preferred: 128 x 256 tiles (twice the operand reuse of 128 x 128), K split so that the SMs are busy; outputs narrower than
// 256 keep 128 x 128 tiles. Returns 0 / 1 when the call does not split.
static int splitk_plan(int layout, int64_t M, int64_t N, int64_t K, int64_t batch, bool plain, bool* wide_out) {
  if (!(layout == FSB_GEMM_TN && batch == 1 && plain && M > 0 && N > 0 && N % 4 == 0 && (M * N) % 8 == 0 && K >= 4096)) return 0;
  const bool wide = N >= 256;
  const int64_t tiles = ((M + GEMM_BM - 1) / GEMM_BM) * (wide ? (N + 255) / 256 : (N + 127) / 128);
  const int64_t slots = num_sms();
  int splits = int(slots / tiles);
  if (splits > 16) splits = 16;
  while (splits > 1 && (K % (int64_t(splits) * GEMM_BK) != 0 || K / splits < 1024)) --splits;
  if (wide_out) *wide_out = wide;
  return (splits >= 2 && tiles * 2 <= slots) ? splits : 0;
}

extern "C" size_t fsb_gemm_workspace_bytes(int layout, int64_t M, int64_t N, int64_t K) {
  const int splits = splitk_plan(layout, M, N, K, 1, true, nullptr);
  return splits ? size_t(splits) * size_t(M) * size_t(N) * sizeof(float) : 0;
}

extern "C" int fsb_gemm_bf16(int layout, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                             int64_t ldb, void* D, int64_t ldd, int d_dtype, const void* bias, int bias_dtype,
                             int epilogue, int accumulate, void* aux, int64_t ldaux, int64_t batch, int64_t stride_a,
                             int64_t stride_b, int64_t stride_d, int64_t stride_aux, void* workspace,
                             size_t workspace_bytes, fsb_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  bool wide = false;
  const int splits = (d_dtype == FSB_BF16 || d_dtype == FSB_F32)
                         ? splitk_plan(layout, M, N, K, batch, bias == nullptr && aux == nullptr && epilogue == FSB_EPI_NONE, &wide)
                         : 0;
  if (splits >= 2) {
    // the scratch is the caller's (fsb_gemm_workspace_bytes): the library allocates nothing. Too small a workspace is an
    // error, not a silent change of algorithm (results would still be correct, but run-to-run timing / rounding would not be
    // what the same call gives with the workspace present).
    const size_t need = size_t(splits) * size_t(M) * size_t(N) * sizeof(float);
    FSB_REQUIRE(workspace != nullptr && workspace_bytes >= need && aligned16(workspace),
                "gemm: this TN call splits K %d ways and needs a %zu-byte workspace (fsb_gemm_workspace_bytes); got %zu",
                splits, need, workspace_bytes);
    {
      float* ws = static_cast<float*>(workspace);
      const int64_t kc = K / splits;
      int rc = gemm_impl(layout, M, N, kc, A, lda, B, ldb, ws, N, FSB_F32, nullptr, FSB_BF16, FSB_EPI_NONE, 0, nullptr, 0,
                         splits, kc * lda, kc * ldb, M * N, 0, stream, wide);
      if (rc) return rc;
      FSB_REQUIRE(ldd % 4 == 0, "gemm: ldd=%ld not vector-aligned", (long)ldd);
      const int64_t work = M * (N / 4);
      const int blocks = int(work / 256 + 1 < 2 * num_sms() ? work / 256 + 1 : 2 * num_sms());
      splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(ws, splits, M, N, D, ldd, d_dtype == FSB_F32, accumulate);
      FSB_CUDA_LAUNCH_CHECK();
      return FSB_OK;
    }
  }
  return gemm_impl(layout, M, N, K, A, lda, B, ldb, D, ldd, d_dtype, bias, bias_dtype, epilogue, accumulate, aux, ldaux, batch,
                   stride_a, stride_b, stride_d, stride_aux, stream);
}

static int fsb::gemm_impl(int layout, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                          int64_t ldb, void* D, int64_t ldd, int d_dtype, const void* bias, int bias_dtype,
                          int epilogue, int accumulate, void* aux, int64_t ldaux, int64_t batch, int64_t stride_a,
                          int64_t stride_b, int64_t stride_d, int64_t stride_aux, cudaStream_t stream, bool force_wide) {
  FSB_REQUIRE(layout >= 0 && layout <= 2, "gemm: bad layout %d", layout);
  FSB_REQUIRE(M > 0 && N > 0 && K > 0 && batch > 0, "gemm: non-positive dims M=%ld N=%ld K=%ld batch=%ld", (long)M,
              (long)N, (long)K, (long)batch);
  FSB_REQUIRE(M < (1 << 30) && N < (1 << 30) && K < (1 << 30), "gemm: dims too large");
  FSB_REQUIRE(A && B && D, "gemm: null operand");
  FSB_REQUIRE(aligned16(A) && aligned16(B) && aligned16(D), "gemm: operands must be 16-byte aligned");
  FSB_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "gemm: lda/ldb must be multiples of 8 (lda=%ld ldb=%ld)", (long)lda,
              (long)ldb);
  FSB_REQUIRE(d_dtype == FSB_BF16 || d_dtype == FSB_F32, "gemm: bad d_dtype");
  FSB_REQUIRE(ldd % (d_dtype == FSB_F32 ? 4 : 8) == 0, "gemm: ldd=%ld not vector-aligned", (long)ldd);
  FSB_REQUIRE(epilogue >= 0 && epilogue <= 2, "gemm: bad epilogue %d", epilogue);
  FSB_REQUIRE(aux == nullptr || (aligned16(aux) && ldaux % 8 == 0), "gemm: aux misaligned");
  FSB_REQUIRE(batch == 1 || (stride_a % 8 == 0 && stride_b % 8 == 0 && stride_d % 8 == 0),
              "gemm: batch strides must be multiples of 8");

  // Tensor maps: always rank 3 (inner, outer, batch).
  CUtensorMap tmA, tmB;
  const bool a_mn = (layout == FSB_GEMM_TN), b_mn = (layout != FSB_GEMM_NT);
  // 128 x 256 tiles unless they would leave a large part of the SMs idle (weight-gradient GEMMs of small models:
  // e.g. 768 x 2304 x 32768 is only 54 such tiles) — then 128 x 128 tiles double the parallelism.
  const int64_t tiles256 = ((M + GEMM_BM - 1) / GEMM_BM) * ((N + 255) / 256) * batch;
  const int BN = (force_wide || (N > 128 && tiles256 * 10 >= int64_t(num_sms()) * 7)) ? 256 : 128;
  {
    // A: K-major -> memory [M rows, K inner]; MN-major -> memory [K rows, M inner]
    uint64_t dims[3] = {uint64_t(a_mn ? M : K), uint64_t(a_mn ? K : M), uint64_t(batch)};
    uint64_t strides[2] = {uint64_t(lda) * 2, uint64_t(batch > 1 ? stride_a : (a_mn ? K : M) * lda) * 2};
    uint32_t box[3] = {64, uint32_t(a_mn ? GEMM_BK : GEMM_BM), 1};
    int rc = make_tmap_bf16(&tmA, A, 3, dims, strides, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {uint64_t(b_mn ? N : K), uint64_t(b_mn ? K : N), uint64_t(batch)};
    uint64_t strides[2] = {uint64_t(ldb) * 2, uint64_t(batch > 1 ? stride_b : (b_mn ? K : N) * ldb) * 2};
    uint32_t box[3] = {64, uint32_t(b_mn ? GEMM_BK : BN), 1};
    int rc = make_tmap_bf16(&tmB, B, 3, dims, strides, box);
    if (rc) return rc;
  }
  GemmParams p;
  p.D = D; p.aux = aux; p.bias = bias;
  p.ldd = ldd; p.ldaux = ldaux; p.stride_d = stride_d; p.stride_aux = stride_aux;
  p.M = int(M); p.N = int(N); p.K = int(K); p.batch = int(batch);
  p.d_f32 = (d_dtype == FSB_F32); p.bias_f32 = (bias_dtype == FSB_F32);
  p.epilogue = epilogue; p.accumulate = accumulate;
  static const int l2hint_env = [] { const char* e = getenv("FSB_GEMM_L2HINT"); return e ? atoi(e) : 0; }();
  p.l2_hints = l2hint_env;
  p.tiles_m = int((M + GEMM_BM - 1) / GEMM_BM);
  p.tiles_n = int((N + BN - 1) / BN);
  // Rasterisation: tiles are walked m-fastest inside groups of group_m m-tiles, so one wave of CTAs touches group_m A panels
  // and #SMs/group_m B panels. HBM traffic per wave is least when both sides weigh about the same (group_m ~ sqrt(#SMs * BN/BM):
  // 16 for 256-wide tiles, 12 for 128-wide ones); the group only grows beyond that while its A panels (group_m x 128 x K bf16)
  // stay well inside the L2 (~32 MB of its 50 MB).
  {
    const int64_t a_panel = int64_t(GEMM_BM) * K * 2;
    const int64_t base = BN == 256 ? 16 : 12;
    int64_t gm = (int64_t(32) << 20) / a_panel;
    gm = gm < base ? base : (gm > 64 ? 64 : gm);
    p.group_m = int(gm);
  }

#define FSB_GEMM_DISPATCH(L) \
  case L:                    \
    return BN == 256 ? launch_gemm<L, 256>(tmA, tmB, p, stream) : launch_gemm<L, 128>(tmA, tmB, p, stream);
  switch (layout) {
    FSB_GEMM_DISPATCH(FSB_GEMM_NT)
    FSB_GEMM_DISPATCH(FSB_GEMM_NN)
    FSB_GEMM_DISPATCH(FSB_GEMM_TN)
  }
#undef FSB_GEMM_DISPATCH
  return FSB_ERR_INVALID;
}
