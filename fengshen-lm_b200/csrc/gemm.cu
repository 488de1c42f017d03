// fsb200 — persistent, warp-specialised bf16 GEMM for sm_90a: TMA -> 128B-swizzled smem -> wgmma (fp32 accumulators in
// registers) -> fused epilogue -> HBM. Replaces the cuBLAS calls behind F.linear on the reference hot path
// (fengshen/models/megatron/mpu/layers.py:347-360, :451-470; layers/transformer.py:136-172) and their autograd
// transposes. Three operand layouts:
//   NT  D = A[M,K] B[N,K]^T   both operands K-major          (forward)
//   NN  D = A[M,K] B[K,N]     B is MN-major in shared memory  (dgrad)
//   TN  D = A[K,M]^T B[K,N]   A and B MN-major                (wgrad)
// MN-major tiles are fetched as 64(mn) x 64(k) TMA boxes; the wgmma descriptor's leading-byte-offset walks the boxes and
// the instruction's transpose bit reads them as MN-major.
//
// Roles (384 threads = 3 warpgroups): warpgroup 0 = TMA producer (one thread issues; setmaxnreg gives its registers to the
// others), warpgroups 1-2 = consumers. Each consumer accumulates 64 rows x BN columns with m64nBNk16 wgmmas and runs the
// epilogue: bias / activation (and the optional accumulate into D) in registers, then 64-row x 128-byte sub-tiles are
// written to a double-buffered, 128B-swizzled shared-memory staging area of its own and leave by TMA bulk stores (D and the
// pre-activation copy alike). The consumer does not wait for a store; it waits only before refilling a staging buffer whose
// previous store has not yet been read out. Ragged tile edges are clipped by the D / aux tensor maps. The producer runs up
// to STAGES k-blocks ahead, across tile boundaries. Grid = min(#tiles, #SMs); static round-robin tile order, grouped for L2.
// Two schedules (gemm_plan picks one per call; each has its own kernel name):
//   cooperative (gemm_bf16_kernel): both consumers work on one 128 x BN tile (BN = 128, 192 or 256), 64 rows each, on the
//     same stages. Long-K and weight-gradient GEMMs.
//   ping-pong (gemm_bf16_pingpong_kernel): each consumer owns whole 64 x 256 tiles and the two take turns on the tensor
//     cores, so one's epilogue runs while the other's mainloop issues MMAs. Short-K GEMMs (K <= 1024), whose 128 x 256
//     epilogue would otherwise leave the tensor cores idle for a visible share of each tile.
// Both issue the same k16 MMA steps per output element in the same order, so the schedule and tile shape never change a bit.
// K-split weight-gradient GEMMs carry the split as the batch coordinate of the tile: split s reads its own range of
// k-blocks of the unbatched operands through full-K tensor maps and writes an fp32 partial product to D[s] (gemm_plan).
#include "gemm_epilogue.cuh"
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
  int ksplits;     // > 1: the batch index is a K-split of unbatched A / B (k_range)
};

// Shared memory: the operand stages, then the epilogue staging area, two 64-row x 128-byte sub-tile buffers (64 bf16 or 32
// fp32 columns) per consumer warpgroup. Double-buffered 8 KB sub-tiles rather than a whole-tile buffer keep all 4 (6) operand
// stages: a 128 x 256 bf16 tile would need 64 KB, i.e. one stage fewer, and the K = 768 GEMMs (12 k-blocks per tile) lean
// on the producer running far ahead across the tile boundary. As many stages as fit, at most 6: 4 for 128 x 256, 128 x 192
// and 64 x 256 tiles, 6 for 128 x 128.
template <int TM, int BN>
struct GemmSmem {
  static constexpr int A_BYTES = TM * GEMM_BK * 2;
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EPI_BUF_BYTES = 64 * 128;
  static constexpr int EPI_BYTES = 2 /*warpgroups*/ * 2 /*buffers*/ * EPI_BUF_BYTES;
  static constexpr int FIT = (kSmemOptIn - 1024 /*align slack*/ - EPI_BYTES - 2 * 6 * 8) / STAGE_BYTES;
  static constexpr int STAGES = FIT < 6 ? FIT : 6;
  static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = EPI_OFFSET + EPI_BYTES;
  // full[STAGES], empty[STAGES]
  static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8 + 1024 /*align slack*/;
  static_assert(TOTAL <= kSmemOptIn, "exceeds the 227 KB of shared memory a block can opt into on sm_90");
};

// K range of a tile: the whole K, or for a K-split GEMM (p.ksplits > 1, batch index = split) the split's share of whole
// k-blocks, [s * nkb / S, (s + 1) * nkb / S). `ab` is the operands' batch coordinate.
__device__ __forceinline__ void k_range(const GemmParams& p, int b, int num_kb, int& kb_lo, int& kb_hi, int& ab) {
  if (p.ksplits > 1) {
    kb_lo = int(int64_t(b) * num_kb / p.ksplits);
    kb_hi = int(int64_t(b + 1) * num_kb / p.ksplits);
    ab = 0;
  } else {
    kb_lo = 0; kb_hi = num_kb; ab = b;
  }
}

// The kernel body. Cooperative (kPP = false): both consumer warpgroups work on one 128 x BN tile, warpgroup wg on rows
// [64 wg, 64 wg + 64), and every stage is read by both. Ping-pong (kPP = true): each warpgroup owns whole TM x BN tiles, the
// CTA's even tiles going to warpgroup 0 and its odd tiles to warpgroup 1, and each stage is read by one warpgroup only. The
// two take turns on the tensor cores: a warpgroup waits for its turn (named barrier 3 + wg), issues its tile's mainloop, and
// hands the turn over (barrier 3 + other) before it drains its MMAs and runs the epilogue, so one warpgroup's epilogue runs
// under the other's mainloop. The turn also keeps the ring sound: a warpgroup only waits on its tile's stages once the other
// has waited on everything before them, so no waiter is ever more than one pass over the ring ahead. The epilogues need no
// ordering of their own: each warpgroup has its own staging buffers and its own TMA store groups.
template <int kLayout, int TM, int BN, bool kPP>
__device__ __forceinline__ void gemm_bf16_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD,
                                               const CUtensorMap& tmAux, const GemmParams& p) {
  constexpr bool A_MN = (kLayout == FSB_GEMM_TN);
  constexpr bool B_MN = (kLayout != FSB_GEMM_NT);
  static_assert(TM == (kPP ? 64 : 128), "each warpgroup accumulates 64 rows of the tile");
  using S = GemmSmem<TM, BN>;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  TmaRing<S::STAGES> ring(reinterpret_cast<uint64_t*>(smem + S::BAR_OFFSET));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.tiles_m * p.tiles_n * p.batch;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    ring.init(kPP ? 4 : 8);
    fence_barrier_init();
  }
  if (threadIdx.x == 128) {
    tma_prefetch_desc(&tmD);
    if (p.aux != nullptr) tma_prefetch_desc(&tmAux);
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer: the CTA's tiles in order, each tile's k-blocks in order =====================
    reg_dec<40>();
    if (threadIdx.x == 0) {
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int b, m_idx, n_idx, kb_lo, kb_hi, ab;
        tile_coords(t, p.tiles_m, p.tiles_n, p.group_m, b, m_idx, n_idx);
        k_range(p, b, num_kb, kb_lo, kb_hi, ab);
        const int m0 = m_idx * TM, n0 = n_idx * BN;
        for (int kb = kb_lo; kb < kb_hi; ++kb) {
          ring.acquire();
          uint8_t* sa = smem + ring.stage * S::STAGE_BYTES;
          uint8_t* sb = sa + S::A_BYTES;
          uint64_t* bar = ring.expect(S::STAGE_BYTES);
          const int k0 = kb * GEMM_BK;
          if constexpr (!A_MN) {
            tma_load_3d(sa, &tmA, bar, k0, m0, ab);
          } else {
#pragma unroll
            for (int c = 0; c < TM / 64; ++c)
              tma_load_3d(sa + c * (GEMM_BK * 128), &tmA, bar, m0 + c * 64, k0, ab);
          }
          if constexpr (!B_MN) {
            tma_load_3d(sb, &tmB, bar, k0, n0, ab);
          } else {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c)
              tma_load_3d(sb + c * (GEMM_BK * 128), &tmB, bar, n0 + c * 64, k0, ab);
          }
          ring.advance();
        }
      }
    }
  } else {
    // ===================== consumers =====================
    reg_inc<232>();  // 256 * 232 + 128 * 40 = 64512
    const int wg = (threadIdx.x >> 7) - 1;
    const int wl = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;   // issues this warpgroup's TMA stores and waits on them
    // The warpgroup's 64 rows of the stage's A: 64 K-major rows or one 64-wide MN-major chunk, 8 KB either way
    const uint32_t a_base = smem_u32(smem) + (kPP ? 0 : wg * 8192);
    const uint64_t dsc_a = A_MN ? make_smem_desc_sw128(a_base, GEMM_BK * 128, 1024) : make_smem_desc_sw128(a_base, 0, 1024);
    const uint64_t dsc_b = B_MN ? make_smem_desc_sw128(smem_u32(smem) + S::A_BYTES, GEMM_BK * 128, 1024)
                                : make_smem_desc_sw128(smem_u32(smem) + S::A_BYTES, 0, 1024);
    uint8_t* const epi_buf = smem + S::EPI_OFFSET + wg * (2 * S::EPI_BUF_BYTES);
    uint32_t n_stored = 0;   // sub-tiles this warpgroup has handed to the TMA unit (selects the staging buffer)
    float acc[BN / 2];
    int i = kPP ? wg : 0;    // the CTA's i-th tile
    for (int t = blockIdx.x + i * gridDim.x; t < num_tiles; t += (kPP ? 2 : 1) * gridDim.x, i += kPP ? 2 : 1) {
      int b, m_idx, n_idx, kb_lo, kb_hi, ab;
      tile_coords(t, p.tiles_m, p.tiles_n, p.group_m, b, m_idx, n_idx);
      k_range(p, b, num_kb, kb_lo, kb_hi, ab);
      if constexpr (kPP) {
        // every tile has num_kb k-blocks (ping-pong runs no K-split): the tile's first stage is the ring's i * num_kb-th
        const int64_t pos = int64_t(i) * num_kb;
        ring.stage = int(pos % S::STAGES);
        ring.phase = uint32_t(pos / S::STAGES) & 1u;
        if (i > 0) bar_sync(3 + wg, 256);   // wait for the turn on the tensor cores
      }
      int prev = 0;
      for (int kb = kb_lo; kb < kb_hi; ++kb) {
        ring.wait();
        const uint64_t so = uint64_t(ring.stage) * (S::STAGE_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) {
          const uint64_t da = dsc_a + so + ((A_MN ? k * 2048 : k * 32) >> 4), db = dsc_b + so + ((B_MN ? k * 2048 : k * 32) >> 4);
          const uint32_t accum = (kb != kb_lo || k != 0) ? 1u : 0u;
          if constexpr (BN == 256) wgmma_ss_n256<A_MN, B_MN>(acc, da, db, accum);
          else if constexpr (BN == 192) wgmma_ss_n192<A_MN, B_MN>(acc, da, db, accum);
          else wgmma_ss_n128<A_MN, B_MN>(acc, da, db, accum);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage can be refilled
        if (kb > kb_lo) ring.release(prev, lane);
        prev = ring.stage;
        ring.advance();
      }
      if constexpr (kPP) {
        if (t + gridDim.x < num_tiles) bar_arrive(3 + (wg ^ 1), 256);   // the other warpgroup's next tile may start
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      ring.release(prev, lane);

      // ---- epilogue: accumulator j covers columns 8 (j / 4) + 2 (lane % 4) + (j & 1), rows r and r + 8 (r = 16 wl + lane / 4)
      const int r = wl * 16 + (lane >> 2);
      const int m0 = m_idx * TM + (kPP ? 0 : 64 * wg), n0 = n_idx * BN;
      const int64_t d_off = int64_t(b) * p.stride_d;
      // One 64-row x 128-byte sub-tile: wait until the store that last used this buffer has read it, fill it, make the
      // writes visible to the async proxy, and hand it to the TMA unit. The consumer never waits for a store to land.
      auto stage_out = [&](const CUtensorMap* tm, int c0, auto&& fill) {
        uint8_t* buf = epi_buf + (n_stored & 1) * S::EPI_BUF_BYTES;
        if (leader) tma_store_wait_read<1>();
        bar_sync(1 + wg, 128);
        fill(buf);
        fence_proxy_async();
        bar_sync(1 + wg, 128);
        if (leader) {
          tma_store_3d(tm, buf, c0, m0, b);
          tma_store_commit();
        }
        ++n_stored;
      };
      // bias (0 without one: the add is kept so that results do not depend on whether a bias was passed)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + 2 * (lane & 3);
        float bv0 = 0.f, bv1 = 0.f;
        if (p.bias != nullptr) {
          if (p.bias_f32) {
            if (col < p.N) bv0 = __ldg(reinterpret_cast<const float*>(p.bias) + col);
            if (col + 1 < p.N) bv1 = __ldg(reinterpret_cast<const float*>(p.bias) + col + 1);
          } else {
            if (col < p.N) bv0 = __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16*>(p.bias) + col));
            if (col + 1 < p.N) bv1 = __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16*>(p.bias) + col + 1));
          }
        }
        acc[4 * j] += bv0; acc[4 * j + 1] += bv1; acc[4 * j + 2] += bv0; acc[4 * j + 3] += bv1;
      }
#pragma unroll
      for (int g = 0; g < BN / 64; ++g) {   // 64 columns = accumulators j in [8 g, 8 g + 8)
        if (p.aux != nullptr) {   // pre-activation copy (bf16)
          stage_out(&tmAux, n0 + 64 * g, [&](uint8_t* buf) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int j = 8 * g + jj;
                *reinterpret_cast<uint32_t*>(buf + swz128(r + 8 * h, 16 * jj + 4 * (lane & 3))) =
                    pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
              }
          });
        }
#pragma unroll
        for (int i = 32 * g; i < 32 * g + 32; ++i) {
          if (p.epilogue == FSB_EPI_GELU_TANH) acc[i] = gelu_tanh_f(acc[i]);
          else if (p.epilogue == FSB_EPI_GELU_ERF) acc[i] = gelu_erf_f(acc[i]);
        }
        if (p.accumulate) {   // D += result: fp32 sum with the old value, rounded once
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * g + jj;
            const int col = n0 + 8 * j + 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = m0 + r + 8 * h;
              if (row >= p.M || col >= p.N) continue;
              const bool two = col + 1 < p.N;
              const int64_t o = d_off + int64_t(row) * p.ldd + col;
              if (p.d_f32) {
                const float* dp = reinterpret_cast<const float*>(p.D) + o;
                if (two) { const float2 q = *reinterpret_cast<const float2*>(dp); acc[4 * j + 2 * h] += q.x; acc[4 * j + 2 * h + 1] += q.y; }
                else acc[4 * j + 2 * h] += *dp;
              } else {
                const __nv_bfloat16* dp = reinterpret_cast<const __nv_bfloat16*>(p.D) + o;
                if (two) { const uint32_t q = *reinterpret_cast<const uint32_t*>(dp); acc[4 * j + 2 * h] += bf16lo(q); acc[4 * j + 2 * h + 1] += bf16hi(q); }
                else acc[4 * j + 2 * h] += __bfloat162float(*dp);
              }
            }
          }
        }
        if (p.d_f32) {   // two 32-column sub-tiles
#pragma unroll
          for (int q = 0; q < 2; ++q)
            stage_out(&tmD, n0 + 64 * g + 32 * q, [&](uint8_t* buf) {
#pragma unroll
              for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int j = 8 * g + 4 * q + jj;
                  *reinterpret_cast<float2*>(buf + swz128(r + 8 * h, 32 * jj + 8 * (lane & 3))) =
                      make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                }
            });
        } else {
          stage_out(&tmD, n0 + 64 * g, [&](uint8_t* buf) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int j = 8 * g + jj;
                *reinterpret_cast<uint32_t*>(buf + swz128(r + 8 * h, 16 * jj + 4 * (lane & 3))) =
                    pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
              }
          });
        }
      }
    }
    if (leader) tma_store_wait<0>();   // every store has completed before the CTA (and its shared memory) goes away
  }
}

// Two entry points so that profiles tell the schedules apart.
template <int kLayout, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmAux, const GemmParams p) {
  gemm_bf16_body<kLayout, GEMM_BM, BN, false>(tmA, tmB, tmD, tmAux, p);
}
template <int kLayout, int TM, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_pingpong_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                          const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmAux,
                          const GemmParams p) {
  gemm_bf16_body<kLayout, TM, BN, true>(tmA, tmB, tmD, tmAux, p);
}

template <int kLayout, int TM, int BN, bool kPP>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD, const CUtensorMap& tmAux,
                       const GemmParams& p, cudaStream_t stream) {
  using S = GemmSmem<TM, BN>;
  const int num_tiles = p.tiles_m * p.tiles_n * p.batch;
  const int grid = num_tiles < gemm_sms() ? num_tiles : gemm_sms();
  if constexpr (kPP) {
    if (int rc = ensure_smem<gemm_bf16_pingpong_kernel<kLayout, TM, BN>>(S::TOTAL, "gemm")) return rc;
    gemm_bf16_pingpong_kernel<kLayout, TM, BN><<<grid, GEMM_THREADS, S::TOTAL, stream>>>(tmA, tmB, tmD, tmAux, p);
  } else {
    if (int rc = ensure_smem<gemm_bf16_kernel<kLayout, BN>>(S::TOTAL, "gemm")) return rc;
    gemm_bf16_kernel<kLayout, BN><<<grid, GEMM_THREADS, S::TOTAL, stream>>>(tmA, tmB, tmD, tmAux, p);
  }
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

// Tile shape, schedule and K-split count.
// - Width: 128 x 256 tiles unless they would leave a large part of the SMs idle (weight-gradient GEMMs of small models: e.g.
//   768 x 2304 x 32768 is only 54 such tiles); then 128 x 128 tiles double the parallelism.
// - K-split: plain, unbatched TN GEMMs (weight gradients) whose output has too few tiles to occupy the SMs (e.g.
//   768 x 768 x 32768: 18 tiles) split K instead: `splits` equal chunks of whole k-blocks, each >= 1024 deep, run as tiles
//   of one launch into an fp32 scratch and are summed in split order (deterministic). Outputs narrower than 256 keep
//   128 x 128 tiles.
// - Ping-pong: an unsplit call that would run 128 x 256 tiles at K <= 1024 runs the ping-pong kernel on 64 x 256 tiles.
//   Short-K tiles spend a visible share of their time in the epilogue (K = 768: 12 k-blocks), which ping-pong hides under
//   the other warpgroup's mainloop. Longer K has less epilogue to hide and keeps the cooperative tile, which loads each B
//   k-block for 128 rows instead of 64. Measured on one H100 80GB HBM3 at 700 W (tools/bench_gemm.py gpt2): 64 x 256
//   ping-pong took c_fc fwd 0.288 -> 0.253 ms and head fwd 4.98 -> 4.63 ms, but c_fc dgrad (K = 3072) 0.223 -> 0.261 and
//   c_attn dgrad (K = 2304) 0.178 -> 0.191; 128 x 128 ping-pong tiles (two m64n128 per k16) were no faster at K = 768
//   (c_fc fwd 0.252, head fwd 4.71 ms) and slower still at K = 3072 (0.304 ms).
// - Wave-aware width: an unsplit TN call on 128 x 128 tiles whose last wave would be less than half full runs 128 x 192
//   tiles if that takes fewer waves (c_fc / mlp_proj wgrad of GPT-2 small on 132 SMs: 144 tiles = 2 waves -> 96 tiles = 1).
// None of these choices changes a result bit: each output element is accumulated by the same k16 MMA steps in the same
// k-block order, and only the K-split (whose count and boundaries these rules leave alone) regroups the sum.
constexpr int GEMM_PP_BM = 64;
constexpr int64_t kPingPongMaxK = 1024;
struct GemmPlan {
  int bn, splits;
  bool pingpong;   // ping-pong kernel on GEMM_PP_BM x bn tiles
};
static GemmPlan gemm_plan(int layout, int64_t M, int64_t N, int64_t K, int64_t batch, bool plain, int sms) {
  const int64_t tiles_m = (M + GEMM_BM - 1) / GEMM_BM;
  const int64_t tiles256 = tiles_m * ((N + 255) / 256) * batch;
  const int bn = (N > 128 && tiles256 * 10 >= int64_t(sms) * 7) ? 256 : 128;
  if (layout == FSB_GEMM_TN && batch == 1 && plain && N % 4 == 0 && (M * N) % 8 == 0 && K >= 4096) {
    const bool wide = N >= 256;
    const int64_t tiles = tiles_m * (wide ? (N + 255) / 256 : (N + 127) / 128);
    int splits = int(sms / tiles);
    if (splits > 16) splits = 16;
    while (splits > 1 && (K % (int64_t(splits) * GEMM_BK) != 0 || K / splits < 1024)) --splits;
    if (splits >= 2 && tiles * 2 <= sms) return {wide ? 256 : bn, splits, false};
  }
  if (bn == 256 && K <= kPingPongMaxK) return {256, 1, true};
  if (bn == 128 && layout == FSB_GEMM_TN && N > 128) {
    const int64_t tiles128 = tiles_m * ((N + 127) / 128) * batch, tiles192 = tiles_m * ((N + 191) / 192) * batch;
    const int64_t last = tiles128 % sms;
    if (last != 0 && last * 2 < sms && (tiles192 + sms - 1) / sms < (tiles128 + sms - 1) / sms) return {192, 1, false};
  }
  return {bn, 1, false};
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
                     int64_t stride_b, int64_t stride_d, int64_t stride_aux, cudaStream_t stream, const GemmPlan& plan);

}  // namespace fsb

using namespace fsb;

extern "C" int fsb_set_reserved_sms(int n) {
  FSB_REQUIRE(n >= 0 && n <= 64, "set_reserved_sms: %d out of range [0, 64]", n);
  fsb::g_reserved_sms = n;
  return FSB_OK;
}

extern "C" size_t fsb_gemm_workspace_bytes(int layout, int64_t M, int64_t N, int64_t K) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  const int splits = gemm_plan(layout, M, N, K, 1, true, gemm_sms()).splits;
  return splits > 1 ? size_t(splits) * size_t(M) * size_t(N) * sizeof(float) : 0;
}

extern "C" int fsb_gemm_bf16(int layout, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                             int64_t ldb, void* D, int64_t ldd, int d_dtype, const void* bias, int bias_dtype,
                             int epilogue, int accumulate, void* aux, int64_t ldaux, int64_t batch, int64_t stride_a,
                             int64_t stride_b, int64_t stride_d, int64_t stride_aux, void* workspace,
                             size_t workspace_bytes, fsb_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  FSB_REQUIRE(M > 0 && N > 0 && K > 0 && batch > 0, "gemm: non-positive dims M=%ld N=%ld K=%ld batch=%ld", (long)M,
              (long)N, (long)K, (long)batch);
  const GemmPlan plan = gemm_plan(layout, M, N, K, batch, bias == nullptr && aux == nullptr && epilogue == FSB_EPI_NONE,
                                  gemm_sms());
  if (plan.splits > 1 && (d_dtype == FSB_BF16 || d_dtype == FSB_F32)) {
    // the scratch is the caller's (fsb_gemm_workspace_bytes): the library allocates nothing. Too small a workspace is an
    // error, not a silent change of algorithm (results would still be correct, but run-to-run timing / rounding would not be
    // what the same call gives with the workspace present).
    const int splits = plan.splits;
    const size_t need = size_t(splits) * size_t(M) * size_t(N) * sizeof(float);
    FSB_REQUIRE(workspace != nullptr && workspace_bytes >= need && aligned16(workspace),
                "gemm: this TN call splits K %d ways and needs a %zu-byte workspace (fsb_gemm_workspace_bytes); got %zu",
                splits, need, workspace_bytes);
    FSB_REQUIRE(ldd % 4 == 0, "gemm: ldd=%ld not vector-aligned", (long)ldd);
    float* ws = static_cast<float*>(workspace);
    // split s: k-blocks k_range(s) of the whole (unbatched) A / B -> fp32 partial ws[s] (M x N, ld N)
    int rc = gemm_impl(layout, M, N, K, A, lda, B, ldb, ws, N, FSB_F32, nullptr, FSB_BF16, FSB_EPI_NONE, 0, nullptr, 0,
                       splits, 0, 0, M * N, 0, stream, GemmPlan{plan.bn, splits, false});
    if (rc) return rc;
    const int64_t work = M * (N / 4);
    const int blocks = int(work / 256 + 1 < 2 * num_sms() ? work / 256 + 1 : 2 * num_sms());
    splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(ws, splits, M, N, D, ldd, d_dtype == FSB_F32, accumulate);
    FSB_CUDA_LAUNCH_CHECK();
    return FSB_OK;
  }
  return gemm_impl(layout, M, N, K, A, lda, B, ldb, D, ldd, d_dtype, bias, bias_dtype, epilogue, accumulate, aux, ldaux, batch,
                   stride_a, stride_b, stride_d, stride_aux, stream, plan);
}

static int fsb::gemm_impl(int layout, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                          int64_t ldb, void* D, int64_t ldd, int d_dtype, const void* bias, int bias_dtype,
                          int epilogue, int accumulate, void* aux, int64_t ldaux, int64_t batch, int64_t stride_a,
                          int64_t stride_b, int64_t stride_d, int64_t stride_aux, cudaStream_t stream,
                          const GemmPlan& plan) {
  const int ksplits = plan.splits;
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
  // D and aux leave through TMA stores, which clip a ragged row end only at 16-byte granularity: an N that ends inside a
  // 16-byte chunk would have the rest of that chunk (columns N.. of the row) overwritten with zeros.
  FSB_REQUIRE(N % (d_dtype == FSB_F32 && aux == nullptr ? 4 : 8) == 0,
              "gemm: N=%ld must be a multiple of %d (8 for a bf16 D or aux, 4 for an fp32 D)", (long)N,
              d_dtype == FSB_F32 && aux == nullptr ? 4 : 8);
  FSB_REQUIRE(epilogue >= 0 && epilogue <= 2, "gemm: bad epilogue %d", epilogue);
  FSB_REQUIRE(aux == nullptr || (aligned16(aux) && ldaux % 8 == 0), "gemm: aux misaligned");
  FSB_REQUIRE(batch == 1 || (stride_a % 8 == 0 && stride_b % 8 == 0 && stride_d % 8 == 0),
              "gemm: batch strides must be multiples of 8");
  FSB_REQUIRE(aux == nullptr || batch == 1 || stride_aux % 8 == 0, "gemm: aux batch stride must be a multiple of 8");
  FSB_REQUIRE(ksplits == 1 || (ksplits > 1 && ksplits <= (K + GEMM_BK - 1) / GEMM_BK && ksplits == batch),
              "gemm: bad K-split count %d", ksplits);

  // Tensor maps: always rank 3 (inner, outer, batch). A K-split GEMM reads unbatched operands and writes D[split].
  CUtensorMap tmA, tmB, tmD, tmAux;
  const bool a_mn = (layout == FSB_GEMM_TN), b_mn = (layout != FSB_GEMM_NT);
  const int BN = plan.bn, TM = plan.pingpong ? GEMM_PP_BM : GEMM_BM;
  const int64_t ab = ksplits > 1 ? 1 : batch;
  {
    // A: K-major -> memory [M rows, K inner]; MN-major -> memory [K rows, M inner]
    uint64_t dims[3] = {uint64_t(a_mn ? M : K), uint64_t(a_mn ? K : M), uint64_t(ab)};
    uint64_t strides[2] = {uint64_t(lda) * 2, uint64_t(ab > 1 ? stride_a : (a_mn ? K : M) * lda) * 2};
    uint32_t box[3] = {64, uint32_t(a_mn ? GEMM_BK : TM), 1};
    int rc = make_tmap_bf16(&tmA, A, 3, dims, strides, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {uint64_t(b_mn ? N : K), uint64_t(b_mn ? K : N), uint64_t(ab)};
    uint64_t strides[2] = {uint64_t(ldb) * 2, uint64_t(ab > 1 ? stride_b : (b_mn ? K : N) * ldb) * 2};
    uint32_t box[3] = {64, uint32_t(b_mn ? GEMM_BK : BN), 1};
    int rc = make_tmap_bf16(&tmB, B, 3, dims, strides, box);
    if (rc) return rc;
  }
  {
    // D / aux: [M rows, N inner], stored as 64-row x 128-byte boxes (64 bf16 or 32 fp32 columns); the map clips ragged edges
    const int64_t es = d_dtype == FSB_F32 ? 4 : 2;
    uint64_t dims[3] = {uint64_t(N), uint64_t(M), uint64_t(batch)};
    uint64_t strides[2] = {uint64_t(ldd * es), uint64_t((batch > 1 ? stride_d : M * ldd) * es)};
    uint32_t box[3] = {uint32_t(128 / es), 64, 1};
    int rc = d_dtype == FSB_F32 ? make_tmap_f32(&tmD, D, 3, dims, strides, box) : make_tmap_bf16(&tmD, D, 3, dims, strides, box);
    if (rc) return rc;
    if (aux != nullptr) {
      uint64_t astrides[2] = {uint64_t(ldaux * 2), uint64_t((batch > 1 ? stride_aux : M * ldaux) * 2)};
      uint32_t abox[3] = {64, 64, 1};
      rc = make_tmap_bf16(&tmAux, aux, 3, dims, astrides, abox);
      if (rc) return rc;
    } else {
      tmAux = tmD;   // never read
    }
  }
  GemmParams p;
  p.D = D; p.aux = aux; p.bias = bias;
  p.ldd = ldd; p.ldaux = ldaux; p.stride_d = stride_d; p.stride_aux = stride_aux;
  p.M = int(M); p.N = int(N); p.K = int(K); p.batch = int(batch);
  p.d_f32 = (d_dtype == FSB_F32); p.bias_f32 = (bias_dtype == FSB_F32);
  p.epilogue = epilogue; p.accumulate = accumulate;
  p.ksplits = ksplits;
  p.tiles_m = int((M + TM - 1) / TM);
  p.tiles_n = int((N + BN - 1) / BN);
  // Rasterisation: tiles are walked m-fastest inside groups of group_m m-tiles, so one wave of CTAs touches group_m A panels
  // and #SMs/group_m B panels. HBM traffic per wave is least when both sides weigh about the same (group_m ~ sqrt(#SMs * BN/TM):
  // 16 for 128 x 256 tiles, 12 for 128 x 128 and 128 x 192, 24 for 64 x 256); the group only grows beyond that while its A
  // panels (group_m x TM x K bf16) stay well inside the L2 (~32 MB of its 50 MB).
  {
    const int64_t a_panel = int64_t(TM) * (K / ksplits) * 2;
    const int64_t base = TM == 64 ? 24 : (BN == 256 ? 16 : 12);
    int64_t gm = (int64_t(32) << 20) / a_panel;
    gm = gm < base ? base : (gm > 64 ? 64 : gm);
    p.group_m = int(gm);
  }

#define FSB_GEMM_DISPATCH(L)                                                                                              \
  case L:                                                                                                                 \
    if (plan.pingpong) return launch_gemm<L, GEMM_PP_BM, 256, true>(tmA, tmB, tmD, tmAux, p, stream);                    \
    if (BN == 256) return launch_gemm<L, GEMM_BM, 256, false>(tmA, tmB, tmD, tmAux, p, stream);                           \
    if (BN == 192 && L == FSB_GEMM_TN) return launch_gemm<FSB_GEMM_TN, GEMM_BM, 192, false>(tmA, tmB, tmD, tmAux, p, stream); \
    return launch_gemm<L, GEMM_BM, 128, false>(tmA, tmB, tmD, tmAux, p, stream);
  switch (layout) {
    FSB_GEMM_DISPATCH(FSB_GEMM_NT)
    FSB_GEMM_DISPATCH(FSB_GEMM_NN)
    FSB_GEMM_DISPATCH(FSB_GEMM_TN)
  }
#undef FSB_GEMM_DISPATCH
  return FSB_ERR_INVALID;
}
