// fsb200 — fused attention backward on wgmma (replaces 3P flash_attn_cuda.bwd called from
// fengshen/models/megatron/layers/flash_attention.py:81-101 and the autograd of the baddbmm/softmax/bmm path,
// transformer.py:307-408; softmax backward formula dx = y*(dy - sum(dy*y)) as in scaled_masked_softmax.h:240-335).
//
// Three launches, all deterministic (no atomics):
//   1. delta[b,h,q] = sum_d dO*O                                   (HBM-bound preprocess)
//   2. dQ kernel : CTA = (b, head, 128 queries), loops over 64-key steps:
//        S = Q K^T, dP = dO V^T (wgmma, fp32 in registers) -> P = exp2(S*c - lse), dS = P*(dP - delta) in registers
//        -> dQ += dS K (dS as the register A operand, K read MN-major from the same shared-memory tile)
//   3. dKV kernel: CTA = (b, head, 128 keys), loops over 64-query steps with the TRANSPOSED products so that a
//        register row is a key row:  S^T = K Q^T, dP^T = V dO^T -> P^T, dS^T -> dV += P^T dO, dK += dS^T Q
//        (dO / Q tiles reused as MN-major B operands; nothing is transposed in memory).
// S and dP are recomputed in both kernels (7 GEMMs instead of 5) — the price of determinism without a dQ reduction.
// Both kernels: warpgroup 0 = TMA producer, warpgroups 1-2 = 64 resident rows each, working on the same streamed stage.
#include "host_common.h"
#include "philox.cuh"
#include "ptx.cuh"

namespace fsb {

constexpr int AB_THREADS = 384;
constexpr int AB_BM = 128;       // rows owned by the CTA (queries for dQ, keys for dKV)
constexpr int AB_BN = 64;        // streamed tile (keys for dQ, queries for dKV)
constexpr int AB_NDIAG = AB_BM + AB_BN - 1;   // diagonals k - q of one 128 x 64 step (bias gradient)
constexpr int AB_DSTRIDE = 192;               // floats per step in the bias-gradient workspace (>= AB_NDIAG)

struct AttBwdParams {
  const float* lse;     // [B,H,Sq] log2 domain
  const float* delta;   // [B,H,Sq]
  const uint8_t* kv_mask;
  const float* rel_bias;     // [nheads, seq_q + seq_kv - 1] additive bias over k - q (natural-log units) or nullptr
  float* dbias_part;         // per-step diagonal sums of dS written by the dQ kernel (see attn_dbias_reduce_kernel)
  __nv_bfloat16 *dq, *dk, *dv;
  int64_t dq_row_stride, dk_row_stride, dv_row_stride, dq_head_stride, dk_head_stride, dv_head_stride;
  int q_head_stride, k_head_stride, v_head_stride, do_head_stride;
  int seq_q, seq_kv, nheads, batch, causal;
  float scale, scale_log2;
  DropArgs drop;             // attention-probability dropout (kDropout only): the forward's seed, stream base and site
  const int *seg_start, *seg_end;   // [batch, seq] segment bounds of each token (kSeg only; see fsb_sdpa_bwd_segments)
};

// ------------------------------------------------------------------------------------------------ delta preprocess
template <int D>
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* __restrict__ o,
                                                         const __nv_bfloat16* __restrict__ dout, float* __restrict__ delta,
                                                         int64_t o_row_stride, int64_t o_head_stride,
                                                         int64_t do_row_stride, int64_t do_head_stride, int batch, int seq,
                                                         int nheads) {
  // one group of D/8 threads per (b, s, h)
  constexpr int G = D / 8;
  const int64_t gid = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) / G;
  const int gl = threadIdx.x % G;
  const int64_t total = int64_t(batch) * seq * nheads;
  float s = 0.f;
  int64_t bs = 0; int h = 0;
  if (gid < total) {
    h = int(gid % nheads);
    bs = gid / nheads;
    float a[8], b[8];
    unpack8(*reinterpret_cast<const uint4*>(o + bs * o_row_stride + h * o_head_stride + gl * 8), a);
    unpack8(*reinterpret_cast<const uint4*>(dout + bs * do_row_stride + h * do_head_stride + gl * 8), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) s += a[j] * b[j];
  }
#pragma unroll
  for (int off = G / 2; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (gid < total && gl == 0) {
    const int64_t b = bs / seq, sq = bs % seq;
    delta[(b * nheads + h) * seq + sq] = s;
  }
}

// ------------------------------------------------------------------------------------------------ shared layout
template <int D, bool kDS>
struct AttBwdSmem {
  static constexpr int BIG_BYTES = AB_BM * D * 2;    // a resident 128-row tile
  static constexpr int SML_BYTES = AB_BN * D * 2;    // a streamed 64-row tile
  static constexpr int STAGES = 3;                   // streamed-tile ring depth
  static constexpr int OFF_BIG0 = 0;                       // dQ: Q     | dKV: K
  static constexpr int OFF_BIG1 = OFF_BIG0 + BIG_BYTES;    // dQ: dO    | dKV: V
  static constexpr int OFF_SML0 = OFF_BIG1 + BIG_BYTES;    // dQ: K_j   | dKV: Q_i   (STAGES)
  static constexpr int OFF_SML1 = OFF_SML0 + STAGES * SML_BYTES;  // dQ: V_j | dKV: dO_i
  static constexpr int OFF_DS = OFF_SML1 + STAGES * SML_BYTES;    // dQ with a bias gradient: fp32 dS tile [128][65]
  static constexpr int OFF_BAR = OFF_DS + (kDS ? (AB_BM * (AB_BN + 1) * 4 + 15) / 16 * 16 : 0);
  static constexpr int NBAR = 1 + 2 * STAGES;  // big_full, sml_full[S], sml_empty[S]
  static constexpr int TOTAL = OFF_BAR + NBAR * 8 + 1024;
  static_assert(TOTAL <= kSmemOptIn, "exceeds the 227 KB of shared memory a block can opt into on sm_90");
};

// shared-memory byte offset of the 16-wide K slice kk of a K-major tile with `rows` rows (64-column swizzle chunks)
__device__ __forceinline__ uint32_t kslice(int kk, int rows) { return (kk / 4) * (rows * 128) + (kk % 4) * 32; }
// 16-key slice kk of a [64 x 64] fp32 accumulator as bf16 register A fragments
__device__ __forceinline__ void to_frag(const float (&x)[32], int kk, uint32_t (&a)[4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = 2 * kk + (r >> 1), h = r & 1;
    a[r] = pack_bf16x2(x[4 * i + 2 * h], x[4 * i + 2 * h + 1]);
  }
}

// ================================================================================================ dQ kernel
// kDropout: dS = P * (dP * Z / (1 - p) - delta), Z regenerated from philox.cuh (delta = rowsum(dO * O) is unchanged).
// kSeg: as in attn_fwd_kernel, the key steps start at seg_start[q0] / AB_BN and each row also masks below its kmin. With
// kDropout, a masked element has P = 0 and so dS = 0 whatever its keep bit, and a visible element's bit does not depend on
// which steps the segment bounds skip (it is a function of its (q, k) only).
// kSeg == kSegBidir: the key steps also stop at ceil(seg_end[last row] / AB_BN), clamped to hold the tile's diagonal step,
// and each row masks above its kmax = seg_end[q] - 1 as well.
template <int D, bool kBias, bool kDropout, int kSeg = kSegNone>
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                   const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                   const AttBwdParams p) {
  using S = AttBwdSmem<D, kBias>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  uint64_t* big_full = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);
  TmaRing<S::STAGES> ring(big_full + 1);   // the streamed tiles

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = gridDim.x - 1 - blockIdx.x;
  const int head = blockIdx.y, b = blockIdx.z;
  const int q0 = tile * AB_BM;
  const int n_all = (p.seq_kv + AB_BN - 1) / AB_BN;
  int n_steps = p.causal ? min(n_all, (min(q0 + AB_BM, p.seq_q) + AB_BN - 1) / AB_BN) : n_all;
  const int* seg_row = kSeg ? p.seg_start + int64_t(b) * p.seq_q : nullptr;
  int j0 = 0;   // first key step, clamped into [0, q0]
  if constexpr (kSeg) j0 = min(max(__ldg(seg_row + q0), 0), q0) / AB_BN;
  const int* end_row = kSeg == kSegBidir ? p.seg_end + int64_t(b) * p.seq_q : nullptr;
  if constexpr (kSeg == kSegBidir) {   // last key step: clamped into [the diagonal step, the last step]
    const int e = min(max(__ldg(end_row + min(q0 + AB_BM, p.seq_q) - 1), 0), p.seq_kv);
    n_steps = min(n_all, max(q0 / AB_BN + 1, (e + AB_BN - 1) / AB_BN));
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmdO); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(big_full, 1);
    ring.init();
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dec<24>();
    if (threadIdx.x == 0) {
      const int qc = head * p.q_head_stride, dc = head * p.do_head_stride;
      const int kc = head * p.k_head_stride, vc = head * p.v_head_stride;
      mbar_expect_tx(big_full, 2 * S::BIG_BYTES);
#pragma unroll
      for (int h = 0; h < D / 64; ++h) {
        tma_load_3d(smem + S::OFF_BIG0 + h * (AB_BM * 128), &tmQ, big_full, qc + h * 64, q0, b);
        tma_load_3d(smem + S::OFF_BIG1 + h * (AB_BM * 128), &tmdO, big_full, dc + h * 64, q0, b);
      }
      for (int j = j0; j < n_steps; ++j) {
        const int st = ring.stage;
        ring.acquire();
        uint64_t* bar = ring.expect(2 * S::SML_BYTES);
#pragma unroll
        for (int h = 0; h < D / 64; ++h) {
          tma_load_3d(smem + S::OFF_SML0 + st * S::SML_BYTES + h * (AB_BN * 128), &tmK, bar, kc + h * 64, j * AB_BN, b);
          tma_load_3d(smem + S::OFF_SML1 + st * S::SML_BYTES + h * (AB_BN * 128), &tmV, bar, vc + h * 64, j * AB_BN, b);
        }
        ring.advance();
      }
    }
    return;
  }

  reg_inc<240>();
  const int wg = (threadIdx.x >> 7) - 1;
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // rows r_lo, r_lo + 8 of the tile
  const int cq = 2 * (lane & 3);
  const uint64_t dsc_q = make_smem_desc_sw128(smem_u32(smem + S::OFF_BIG0) + wg * (64 * 128), 0, 1024);
  const uint64_t dsc_do = make_smem_desc_sw128(smem_u32(smem + S::OFF_BIG1) + wg * (64 * 128), 0, 1024);
  const uint64_t dsc_k = make_smem_desc_sw128(smem_u32(smem + S::OFF_SML0), 0, 1024);              // K-major view (S)
  const uint64_t dsc_v = make_smem_desc_sw128(smem_u32(smem + S::OFF_SML1), 0, 1024);
  const uint64_t dsc_kmn = make_smem_desc_sw128(smem_u32(smem + S::OFF_SML0), AB_BN * 128, 1024);  // MN-major view (dQ)
  const uint8_t* mrow = p.kv_mask ? p.kv_mask + int64_t(b) * p.seq_kv : nullptr;
  const int n_rel = p.seq_q + p.seq_kv - 1;
  int q_row[2], kmax[2], kmin[2] = {0, 0};
  float lse[2], delta[2];
  const float* brow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    q_row[h] = q0 + r_lo + 8 * h;
    const bool ok = q_row[h] < p.seq_q;
    const int64_t si = (int64_t(b) * p.nheads + head) * p.seq_q + q_row[h];
    lse[h] = ok ? p.lse[si] : INFINITY;
    delta[h] = ok ? p.delta[si] : 0.f;
    kmax[h] = p.causal ? min(q_row[h], p.seq_kv - 1) : p.seq_kv - 1;   // last key column this row may attend to
    if constexpr (kSeg) kmin[h] = ok ? __ldg(seg_row + q_row[h]) : 0;   // first one
    if constexpr (kSeg == kSegBidir) kmax[h] = ok ? min(__ldg(end_row + q_row[h]) - 1, kmax[h]) : kmax[h];
    // relative-position bias (mT5): this row reads entries (k - q_row + seq_q - 1) of its head's vector
    brow[h] = kBias ? p.rel_bias + int64_t(head) * n_rel + (p.seq_q - 1 - min(q_row[h], p.seq_q - 1)) : nullptr;
  }
  float* dpart = kBias && p.dbias_part ? p.dbias_part + ((int64_t(b) * p.nheads + head) * gridDim.x + tile) * n_all * AB_DSTRIDE
                                       : nullptr;
  float dq[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dq[i] = 0.f;
  DropKey dkey;
  if constexpr (kDropout) dkey = drop_key(p.drop);

  mbar_wait(big_full, 0);
  for (int j = j0; j < n_steps; ++j) {
    const auto step = ring.at(j - j0);
    const uint64_t sto = uint64_t(step.stage) * (S::SML_BYTES >> 4);
    float s[32], dp[32];
    step.wait();
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss_n64<0, 0>(s, dsc_q + (kslice(kk, AB_BM) >> 4), dsc_k + sto + (kslice(kk, AB_BN) >> 4), kk != 0 ? 1u : 0u);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss_n64<0, 0>(dp, dsc_do + (kslice(kk, AB_BM) >> 4), dsc_v + sto + (kslice(kk, AB_BN) >> 4), kk != 0 ? 1u : 0u);
    wgmma_commit();
    const int c0 = j * AB_BN;
    uint32_t dw[kDropout ? AB_BN / 16 : 1][2];   // the forward's keep bits, regenerated while the tensor cores work
    if constexpr (kDropout) attn_drop_rows<AB_BN / 16>(dkey, uint32_t(b * p.nheads + head), q0 + r_lo, c0, lane, dw);
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    wgmma_fence_acc(dp);
    bool need_mask = (p.causal && c0 + AB_BN - 1 > q0 + wg * 64) || (c0 + AB_BN > p.seq_kv) || mrow ||
                     (kSeg && c0 < max(kmin[0], kmin[1]));
    if constexpr (kSeg == kSegBidir) need_mask = need_mask || c0 + AB_BN - 1 > min(kmax[0], kmax[1]);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int h = e >> 1, col = c0 + 8 * i + cq + (e & 1);
        float x = s[4 * i + e] * p.scale_log2 - lse[h];
        if constexpr (kBias) x = fmaf(__ldg(brow[h] + min(col, p.seq_kv - 1)), 1.4426950408889634f, x);
        float pe = ex2_approx(x);
        if (need_mask) {
          bool keep = col <= kmax[h];
          if constexpr (kSeg) keep = keep && col >= kmin[h];
          if (mrow != nullptr && keep) keep = mrow[col] != 0;
          pe = keep ? pe : 0.f;
        }
        float dpe = dp[4 * i + e];
        if constexpr (kDropout) dpe = drop_keep(dw[i >> 1][e & 1], 2 * h + (i & 1), dkey.thr) ? dpe * p.drop.keep_scale : 0.f;
        s[4 * i + e] = pe * (dpe - delta[h]);   // dS
      }
    }
    if constexpr (kBias) {
      // Bias gradient: dBias[h, k - q] = sum of dS over each diagonal. The step's 128 x 64 dS tile goes to shared memory and
      // thread t sums diagonal t - 127 of it in row order into its own slot of the workspace (plain stores, no atomics);
      // attn_dbias_reduce_kernel adds the slots up in a fixed order.
      if (dpart != nullptr) {
        float* tds = reinterpret_cast<float*>(smem + S::OFF_DS);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) tds[(r_lo + 8 * (e >> 1)) * (AB_BN + 1) + 8 * i + cq + (e & 1)] = s[4 * i + e];
        bar_sync(1, 256);
        const int t = threadIdx.x - 128;
        if (t < AB_NDIAG) {
          const int o = t - (AB_BM - 1);
          float acc = 0.f;
          for (int r = max(0, -o); r < min(AB_BM, AB_BN - o); ++r) acc += tds[r * (AB_BN + 2) + o];
          dpart[int64_t(j) * AB_DSTRIDE + t] = acc;
        }
        bar_sync(1, 256);
      }
    }
    uint32_t a[AB_BN / 16][4];
#pragma unroll
    for (int kk = 0; kk < AB_BN / 16; ++kk) to_frag(s, kk, a[kk]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_BN / 16; ++kk) wgmma_rs_dim<D, 1>(dq, a[kk], dsc_kmn + sto + ((kk * 2048) >> 4), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dq);
    __syncwarp();
    step.release(lane);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (q_row[h] >= p.seq_q) continue;
    __nv_bfloat16* dqp = p.dq + (int64_t(b) * p.seq_q + q_row[h]) * p.dq_row_stride + int64_t(head) * p.dq_head_stride + cq;
#pragma unroll
    for (int i = 0; i < D / 8; ++i)
      *reinterpret_cast<uint32_t*>(dqp + 8 * i) = pack_bf16x2(dq[4 * i + 2 * h] * p.scale, dq[4 * i + 2 * h + 1] * p.scale);
  }
}

// ================================================================================================ dK / dV kernel
// kDropout: dV += (P * Z / (1 - p))^T dO and dS^T = P^T * (dP^T * Z / (1 - p) - delta); a register row is a key row here, so
// the mask comes from attn_drop_cols (same Philox calls as the row-major kernels, words picked along the other axis).
// kSeg: key k is seen by the queries k <= q < seg_end[k]. The tile's last key has the largest end, so the query steps stop at
// ceil(seg_end[last key] / AB_BN) (clamped into the sequence); each key row masks above its qmax = seg_end[k] - 1. With
// kDropout the segment mask zeroes P^T before the keep bits scale it, so both dV and dS^T are 0 past qmax whatever the bit.
// kSeg == kSegBidir: key k is seen by the queries seg_start[k] <= q < seg_end[k]. The tile's first key has the smallest start,
// so the query steps run from seg_start[first key] / AB_BN to ceil(seg_end[last key] / AB_BN), clamped into the sequence and
// to hold the tile's diagonal steps; a step masks when it crosses a row's qmin = seg_start[k] or its qmax.
template <int D, bool kBias, bool kDropout, int kSeg = kSegNone>
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmdO,
                    const AttBwdParams p) {
  using S = AttBwdSmem<D, false>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  uint64_t* big_full = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);
  TmaRing<S::STAGES> ring(big_full + 1);   // the streamed tiles

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x;  // early key tiles see the most queries under a causal mask: they come first already
  const int head = blockIdx.y, b = blockIdx.z;
  const int kv0 = tile * AB_BM;
  const int n_q = (p.seq_q + AB_BN - 1) / AB_BN;
  int i_start = p.causal ? min(n_q, kv0 / AB_BN) : 0;
  const int* seg_row = kSeg ? p.seg_end + int64_t(b) * p.seq_kv : nullptr;
  int i_end = n_q;
  if constexpr (kSeg) i_end = min(n_q, (min(max(__ldg(seg_row + min(kv0 + AB_BM, p.seq_kv) - 1), 0), p.seq_q) + AB_BN - 1) / AB_BN);
  const int* start_row = kSeg == kSegBidir ? p.seg_start + int64_t(b) * p.seq_kv : nullptr;
  if constexpr (kSeg == kSegBidir) {   // first query step clamped into [0, kv0]; the last at least the diagonal step
    i_start = min(max(__ldg(start_row + kv0), 0), kv0) / AB_BN;
    i_end = min(n_q, max(i_end, kv0 / AB_BN + 1));
  }
  const int n_steps = kSeg ? max(0, i_end - i_start) : n_q - i_start;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmdO); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(big_full, 1);
    ring.init();
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dec<24>();
    if (threadIdx.x == 0) {
      const int qc = head * p.q_head_stride, dc = head * p.do_head_stride;
      const int kc = head * p.k_head_stride, vc = head * p.v_head_stride;
      mbar_expect_tx(big_full, 2 * S::BIG_BYTES);
#pragma unroll
      for (int h = 0; h < D / 64; ++h) {
        tma_load_3d(smem + S::OFF_BIG0 + h * (AB_BM * 128), &tmK, big_full, kc + h * 64, kv0, b);
        tma_load_3d(smem + S::OFF_BIG1 + h * (AB_BM * 128), &tmV, big_full, vc + h * 64, kv0, b);
      }
      for (int i = 0; i < n_steps; ++i) {
        const int st = ring.stage;
        ring.acquire();
        uint64_t* bar = ring.expect(2 * S::SML_BYTES);
#pragma unroll
        for (int h = 0; h < D / 64; ++h) {
          tma_load_3d(smem + S::OFF_SML0 + st * S::SML_BYTES + h * (AB_BN * 128), &tmQ, bar, qc + h * 64, (i_start + i) * AB_BN, b);
          tma_load_3d(smem + S::OFF_SML1 + st * S::SML_BYTES + h * (AB_BN * 128), &tmdO, bar, dc + h * 64, (i_start + i) * AB_BN, b);
        }
        ring.advance();
      }
    }
    return;
  }

  reg_inc<240>();
  const int wg = (threadIdx.x >> 7) - 1;
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // key rows r_lo, r_lo + 8 of the tile
  const int cq = 2 * (lane & 3);
  const uint64_t dsc_k = make_smem_desc_sw128(smem_u32(smem + S::OFF_BIG0) + wg * (64 * 128), 0, 1024);
  const uint64_t dsc_v = make_smem_desc_sw128(smem_u32(smem + S::OFF_BIG1) + wg * (64 * 128), 0, 1024);
  const uint64_t dsc_q = make_smem_desc_sw128(smem_u32(smem + S::OFF_SML0), 0, 1024);               // K-major view (S^T)
  const uint64_t dsc_do = make_smem_desc_sw128(smem_u32(smem + S::OFF_SML1), 0, 1024);
  const uint64_t dsc_qmn = make_smem_desc_sw128(smem_u32(smem + S::OFF_SML0), AB_BN * 128, 1024);   // MN-major view (dK)
  const uint64_t dsc_domn = make_smem_desc_sw128(smem_u32(smem + S::OFF_SML1), AB_BN * 128, 1024);  // MN-major view (dV)
  const int64_t stat_base = (int64_t(b) * p.nheads + head) * p.seq_q;
  const int n_rel = p.seq_q + p.seq_kv - 1;
  int kv_row[2];
  bool row_ok[2];
  const float* bkey[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    kv_row[h] = kv0 + r_lo + 8 * h;
    row_ok[h] = kv_row[h] < p.seq_kv && (p.kv_mask == nullptr || p.kv_mask[int64_t(b) * p.seq_kv + kv_row[h]] != 0);
    // relative-position bias: key row kv_row, query column qi -> entry (kv_row - qi + seq_q - 1) of the head's vector
    bkey[h] = kBias ? p.rel_bias + int64_t(head) * n_rel + (min(kv_row[h], p.seq_kv - 1) + p.seq_q - 1) : nullptr;
  }
  // kSeg: the tile's first key has the smallest qmax (last query seeing it). Only the steps past it mask, and they re-read
  // their rows' qmax from global memory: two more live registers would spill in the D = 128 kernel.
  int qlim = 0;
  if constexpr (kSeg) qlim = __ldg(seg_row + kv0) - 1;
  // kSegBidir: likewise the tile's last key has the largest qmin; only the steps before it mask below, re-reading their rows'
  // qmin (both bounds live in registers would cost a spill)
  int qlo = 0;
  if constexpr (kSeg == kSegBidir) qlo = __ldg(start_row + min(kv0 + AB_BM, p.seq_kv) - 1);
  float dv[D / 2], dk[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  DropKey dkey;
  if constexpr (kDropout) dkey = drop_key(p.drop);

  mbar_wait(big_full, 0);
  for (int i = 0; i < n_steps; ++i) {
    const auto step = ring.at(i);
    const uint64_t sto = uint64_t(step.stage) * (S::SML_BYTES >> 4);
    const int qt0 = (i_start + i) * AB_BN;
    float s[32], dp[32];
    step.wait();
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss_n64<0, 0>(s, dsc_k + (kslice(kk, AB_BM) >> 4), dsc_q + sto + (kslice(kk, AB_BN) >> 4), kk != 0 ? 1u : 0u);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss_n64<0, 0>(dp, dsc_v + (kslice(kk, AB_BM) >> 4), dsc_do + sto + (kslice(kk, AB_BN) >> 4), kk != 0 ? 1u : 0u);
    wgmma_commit();
    // the forward's keep bits, regenerated while the tensor cores work; one bit per element, so a single register carries
    // them past the wait
    uint32_t zbits = 0;
    if constexpr (kDropout) zbits = attn_keep_cols<AB_BN / 16>(dkey, uint32_t(b * p.nheads + head), kv0 + r_lo, qt0, lane);
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    wgmma_fence_acc(dp);
    const bool need_causal = p.causal && (qt0 < kv0 + AB_BM - 1);
    const bool need_seg = kSeg && qt0 + AB_BN - 1 > qlim;
    int qmax[2] = {0, 0};
    if (need_seg) {
#pragma unroll
      for (int h = 0; h < 2; ++h) qmax[h] = row_ok[h] ? __ldg(p.seg_end + int64_t(b) * p.seq_kv + kv_row[h]) - 1 : -1;
    }
    const bool need_lo = kSeg == kSegBidir && qt0 < qlo;
    int qmin[2] = {0, 0};
    if constexpr (kSeg == kSegBidir) {
      if (need_lo) {
#pragma unroll
        for (int h = 0; h < 2; ++h) qmin[h] = row_ok[h] ? __ldg(start_row + kv_row[h]) : 0;
      }
    }
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int qi = qt0 + 8 * ii + cq + c;
        const bool q_ok = qi < p.seq_q;
        const float lse_c = q_ok ? __ldg(p.lse + stat_base + qi) : INFINITY;
        const float del_c = q_ok ? __ldg(p.delta + stat_base + qi) : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int e = 2 * h + c;
          float arg = s[4 * ii + e] * p.scale_log2 - lse_c;
          if constexpr (kBias) arg = fmaf(__ldg(bkey[h] - min(qi, p.seq_q - 1)), 1.4426950408889634f, arg);
          float x = ex2_approx(arg);
          bool keep = row_ok[h] && !(need_causal && qi < kv_row[h]) && !(need_seg && qi > qmax[h]);
          if constexpr (kSeg == kSegBidir) keep = keep && !(need_lo && qi < qmin[h]);
          x = keep ? x : 0.f;
          if constexpr (kDropout) {
            const bool z = (zbits >> (4 * ii + e)) & 1u;
            s[4 * ii + e] = z ? x * p.drop.keep_scale : 0.f;                                    // (P * Z / (1 - p))^T
            dp[4 * ii + e] = x * ((z ? dp[4 * ii + e] * p.drop.keep_scale : 0.f) - del_c);      // dS^T
          } else {
            s[4 * ii + e] = x;                                  // P^T
            dp[4 * ii + e] = x * (dp[4 * ii + e] - del_c);      // dS^T
          }
        }
      }
    }
    uint32_t pa[AB_BN / 16][4], da[AB_BN / 16][4];
#pragma unroll
    for (int kk = 0; kk < AB_BN / 16; ++kk) { to_frag(s, kk, pa[kk]); to_frag(dp, kk, da[kk]); }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_BN / 16; ++kk) wgmma_rs_dim<D, 1>(dv, pa[kk], dsc_domn + sto + ((kk * 2048) >> 4), 1u);
#pragma unroll
    for (int kk = 0; kk < AB_BN / 16; ++kk) wgmma_rs_dim<D, 1>(dk, da[kk], dsc_qmn + sto + ((kk * 2048) >> 4), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dv);
    wgmma_fence_acc(dk);
    __syncwarp();
    step.release(lane);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (kv_row[h] >= p.seq_kv) continue;
    __nv_bfloat16* dvp = p.dv + (int64_t(b) * p.seq_kv + kv_row[h]) * p.dv_row_stride + int64_t(head) * p.dv_head_stride + cq;
    __nv_bfloat16* dkp = p.dk + (int64_t(b) * p.seq_kv + kv_row[h]) * p.dk_row_stride + int64_t(head) * p.dk_head_stride + cq;
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      *reinterpret_cast<uint32_t*>(dvp + 8 * i) = pack_bf16x2(dv[4 * i + 2 * h], dv[4 * i + 2 * h + 1]);
      *reinterpret_cast<uint32_t*>(dkp + 8 * i) = pack_bf16x2(dk[4 * i + 2 * h] * p.scale, dk[4 * i + 2 * h + 1] * p.scale);
    }
  }
}

// dBias[h, i] (+)= sum over (b, q tile, step) of the diagonal sums the dQ kernel left in the workspace, in a FIXED order
// (deterministic). i = (k - q) + seq_q - 1. Stage 1: grid (i chunks, heads, batch splits) -> part2[split][h][i]; stage 2 adds
// the splits onto the caller's fp32 vector.
__global__ void __launch_bounds__(128) attn_dbias_reduce_kernel(const float* __restrict__ part, float* __restrict__ part2,
                                                                int batch, int nheads, int seq_q, int seq_kv, int causal,
                                                                int n_qtiles, int bsplit) {
  const int n_rel = seq_q + seq_kv - 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int h = blockIdx.y, sp = blockIdx.z;
  if (i >= n_rel) return;
  const int d = i - (seq_q - 1);
  const int n_all = (seq_kv + AB_BN - 1) / AB_BN;
  const int b0 = int(int64_t(batch) * sp / bsplit), b1 = int(int64_t(batch) * (sp + 1) / bsplit);
  float acc = 0.f;
  for (int b = b0; b < b1; ++b) {
    for (int tile = 0; tile < n_qtiles; ++tile) {
      const int q0 = tile * AB_BM;
      const int n_steps = causal ? min(n_all, (min(q0 + AB_BM, seq_q) + AB_BN - 1) / AB_BN) : n_all;
      const float* base = part + ((int64_t(b) * nheads + h) * n_qtiles + tile) * n_all * AB_DSTRIDE;
      // step j holds the diagonal k - q = d in slot t = d + q0 - 64 j + 127 when 0 <= t < 191
      const int hi = d + q0 + (AB_BM - 1), lo = d + q0 - (AB_BN - 1);
      if (hi < 0) continue;
      const int j_lo = lo <= 0 ? 0 : (lo + AB_BN - 1) / AB_BN, j_hi = min(n_steps - 1, hi / AB_BN);
      for (int j = j_lo; j <= j_hi; ++j) acc += base[int64_t(j) * AB_DSTRIDE + (hi - j * AB_BN)];
    }
  }
  part2[(int64_t(sp) * nheads + h) * n_rel + i] = acc;
}
__global__ void __launch_bounds__(128) attn_dbias_final_kernel(const float* __restrict__ part2, float* __restrict__ dbias,
                                                               int nheads, int n_rel, int bsplit) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int h = blockIdx.y;
  if (i >= n_rel) return;
  float acc = dbias[int64_t(h) * n_rel + i];
  for (int sp = 0; sp < bsplit; ++sp) acc += part2[(int64_t(sp) * nheads + h) * n_rel + i];
  dbias[int64_t(h) * n_rel + i] = acc;
}
static inline int dbias_bsplit(int batch) { return batch < 16 ? batch : 16; }
static inline size_t dbias_part_floats(int64_t batch, int64_t seq_q, int64_t seq_kv, int nheads) {
  const int64_t n_qt = (seq_q + AB_BM - 1) / AB_BM, n_all = (seq_kv + AB_BN - 1) / AB_BN;
  return size_t(batch) * nheads * n_qt * n_all * AB_DSTRIDE;
}

template <int D, bool kBias, bool kDropout, int kSeg = kSegNone>
static int launch_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout,
                           int64_t q_rs, int64_t k_rs, int64_t v_rs, int64_t o_rs, int64_t do_rs, int64_t o_hs,
                           float* delta, AttBwdParams& p, float* drel_bias, float* part2, cudaStream_t st) {
  using SQ = AttBwdSmem<D, kBias>;
  using SK = AttBwdSmem<D, false>;
  if (int rc = ensure_smem<attn_bwd_dq_kernel<D, kBias, kDropout, kSeg>>(SQ::TOTAL, "sdpa_bwd")) return rc;
  if (int rc = ensure_smem<attn_bwd_dkv_kernel<D, kBias, kDropout, kSeg>>(SK::TOTAL, "sdpa_bwd")) return rc;
  // 1. delta
  {
    const int64_t groups = int64_t(p.batch) * p.seq_q * p.nheads;
    const int64_t threads = groups * (D / 8);
    attn_delta_kernel<D><<<unsigned((threads + 255) / 256), 256, 0, st>>>(
        (const __nv_bfloat16*)o, (const __nv_bfloat16*)dout, delta, o_rs, o_hs, do_rs, p.do_head_stride, p.batch, p.seq_q,
        p.nheads);
    FSB_CUDA_LAUNCH_CHECK();
  }
  CUtensorMap tq128, tdo128, tk64, tv64, tk128, tv128, tq64, tdo64;
  int rc;
  const int64_t wq = int64_t(p.nheads - 1) * p.q_head_stride + D, wk = int64_t(p.nheads - 1) * p.k_head_stride + D;
  const int64_t wv = int64_t(p.nheads - 1) * p.v_head_stride + D, wdo = int64_t(p.nheads - 1) * p.do_head_stride + D;
  if ((rc = make_attn_tmap(&tq128, q, q_rs, wq, p.seq_q, p.batch, AB_BM))) return rc;
  if ((rc = make_attn_tmap(&tdo128, dout, do_rs, wdo, p.seq_q, p.batch, AB_BM))) return rc;
  if ((rc = make_attn_tmap(&tk64, k, k_rs, wk, p.seq_kv, p.batch, AB_BN))) return rc;
  if ((rc = make_attn_tmap(&tv64, v, v_rs, wv, p.seq_kv, p.batch, AB_BN))) return rc;
  if ((rc = make_attn_tmap(&tk128, k, k_rs, wk, p.seq_kv, p.batch, AB_BM))) return rc;
  if ((rc = make_attn_tmap(&tv128, v, v_rs, wv, p.seq_kv, p.batch, AB_BM))) return rc;
  if ((rc = make_attn_tmap(&tq64, q, q_rs, wq, p.seq_q, p.batch, AB_BN))) return rc;
  if ((rc = make_attn_tmap(&tdo64, dout, do_rs, wdo, p.seq_q, p.batch, AB_BN))) return rc;
  // 2. dQ
  {
    dim3 grid((p.seq_q + AB_BM - 1) / AB_BM, p.nheads, p.batch);
    attn_bwd_dq_kernel<D, kBias, kDropout, kSeg><<<grid, AB_THREADS, SQ::TOTAL, st>>>(tq128, tdo128, tk64, tv64, p);
    FSB_CUDA_LAUNCH_CHECK();
    if (kBias && drel_bias != nullptr) {
      const int n_rel = p.seq_q + p.seq_kv - 1, bs = dbias_bsplit(p.batch);
      attn_dbias_reduce_kernel<<<dim3((n_rel + 127) / 128, p.nheads, bs), 128, 0, st>>>(
          p.dbias_part, part2, p.batch, p.nheads, p.seq_q, p.seq_kv, p.causal, int(grid.x), bs);
      FSB_CUDA_LAUNCH_CHECK();
      attn_dbias_final_kernel<<<dim3((n_rel + 127) / 128, p.nheads), 128, 0, st>>>(part2, drel_bias, p.nheads, n_rel, bs);
      FSB_CUDA_LAUNCH_CHECK();
    }
  }
  // 3. dK, dV
  {
    dim3 grid((p.seq_kv + AB_BM - 1) / AB_BM, p.nheads, p.batch);
    attn_bwd_dkv_kernel<D, kBias, kDropout, kSeg><<<grid, AB_THREADS, SK::TOTAL, st>>>(tk128, tv128, tq64, tdo64, p);
    FSB_CUDA_LAUNCH_CHECK();
  }
  return FSB_OK;
}

}  // namespace fsb

using namespace fsb;

static int sdpa_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                    float* delta, void* dq, void* dk, void* dv, int64_t batch, int64_t seq_q, int64_t seq_kv, int nheads,
                    int head_dim, int64_t q_row_stride, int64_t k_row_stride, int64_t v_row_stride, int64_t o_row_stride,
                    int64_t do_row_stride, int64_t dq_row_stride, int64_t dk_row_stride, int64_t dv_row_stride,
                    int64_t q_head_stride, int64_t k_head_stride, int64_t v_head_stride, int64_t o_head_stride,
                    int64_t do_head_stride, int64_t dq_head_stride, int64_t dk_head_stride, int64_t dv_head_stride,
                    float scale, int causal, const uint8_t* kv_mask, const float* rel_bias, float* drel_bias,
                    void* workspace, size_t workspace_bytes, const DropArgs* drop, const int* seg_start,
                    const int* seg_end, fsb_stream_t st) {
  FSB_REQUIRE(q && k && v && o && dout && lse && delta && dq && dk && dv, "sdpa_bwd: null pointer");
  FSB_REQUIRE(head_dim == 64 || head_dim == 128, "sdpa_bwd: head_dim %d unsupported (64 or 128)", head_dim);
  FSB_REQUIRE(batch > 0 && seq_q > 0 && seq_kv > 0 && nheads > 0 && batch < 65536 && nheads < 65536, "sdpa_bwd: bad dims");
  FSB_REQUIRE(!causal || seq_q == seq_kv, "sdpa_bwd: causal needs seq_q == seq_kv");
  FSB_REQUIRE(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(o) && aligned16(dout) && aligned16(dq) &&
                  aligned16(dk) && aligned16(dv),
              "sdpa_bwd: 16-byte alignment required");
  FSB_REQUIRE((q_row_stride | k_row_stride | v_row_stride | o_row_stride | do_row_stride | dq_row_stride |
               dk_row_stride | dv_row_stride | q_head_stride | k_head_stride | v_head_stride | o_head_stride |
               do_head_stride | dq_head_stride | dk_head_stride | dv_head_stride) % 8 == 0,
              "sdpa_bwd: strides must be multiples of 8 elements");
  FSB_REQUIRE(drel_bias == nullptr || rel_bias != nullptr, "sdpa_bwd: drel_bias without rel_bias");
  AttBwdParams p;
  p.lse = lse; p.delta = delta; p.kv_mask = kv_mask;
  p.rel_bias = rel_bias; p.dbias_part = nullptr;
  float* part2 = nullptr;
  if (drel_bias != nullptr) {
    const size_t need = fsb_sdpa_bwd_workspace_bytes(batch, seq_q, seq_kv, nheads);
    FSB_REQUIRE(workspace != nullptr && workspace_bytes >= need && aligned16(workspace),
                "sdpa_bwd: the bias gradient needs a %zu-byte workspace (fsb_sdpa_bwd_workspace_bytes); got %zu", need,
                workspace_bytes);
    p.dbias_part = static_cast<float*>(workspace);
    part2 = p.dbias_part + dbias_part_floats(batch, seq_q, seq_kv, nheads);
  }
  p.dq = (__nv_bfloat16*)dq; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv;
  p.dq_row_stride = dq_row_stride; p.dk_row_stride = dk_row_stride; p.dv_row_stride = dv_row_stride;
  p.dq_head_stride = dq_head_stride; p.dk_head_stride = dk_head_stride; p.dv_head_stride = dv_head_stride;
  p.q_head_stride = int(q_head_stride); p.k_head_stride = int(k_head_stride); p.v_head_stride = int(v_head_stride);
  p.do_head_stride = int(do_head_stride);
  p.seq_q = int(seq_q); p.seq_kv = int(seq_kv); p.nheads = nheads; p.batch = int(batch); p.causal = causal;
  p.scale = scale; p.scale_log2 = scale * 1.4426950408889634f;
  p.seg_start = seg_start; p.seg_end = seg_end;
  if (seg_start != nullptr && !causal) {   // fsb_sdpa_bwd_segments_bidirectional: head_dim 64, no bias, no key mask
    if (drop != nullptr) {
      p.drop = *drop;
      return launch_attn_bwd<64, false, true, kSegBidir>(q, k, v, o, dout, q_row_stride, k_row_stride, v_row_stride,
                                                         o_row_stride, do_row_stride, o_head_stride, delta, p, nullptr,
                                                         nullptr, (cudaStream_t)st);
    }
    return launch_attn_bwd<64, false, false, kSegBidir>(q, k, v, o, dout, q_row_stride, k_row_stride, v_row_stride,
                                                        o_row_stride, do_row_stride, o_head_stride, delta, p, nullptr,
                                                        nullptr, (cudaStream_t)st);
  }
  if (seg_start != nullptr && drop != nullptr) {   // fsb_sdpa_bwd_segments_dropout with p > 0: head_dim 64 only
    p.drop = *drop;
    return launch_attn_bwd<64, false, true, kSegCausal>(q, k, v, o, dout, q_row_stride, k_row_stride, v_row_stride, o_row_stride,
                                                  do_row_stride, o_head_stride, delta, p, nullptr, nullptr, (cudaStream_t)st);
  }
  if (seg_start != nullptr)   // fsb_sdpa_bwd_segments: causal, no bias, no dropout, no key mask
    return head_dim == 128
               ? launch_attn_bwd<128, false, false, kSegCausal>(q, k, v, o, dout, q_row_stride, k_row_stride, v_row_stride,
                                                          o_row_stride, do_row_stride, o_head_stride, delta, p, nullptr,
                                                          nullptr, (cudaStream_t)st)
               : launch_attn_bwd<64, false, false, kSegCausal>(q, k, v, o, dout, q_row_stride, k_row_stride, v_row_stride,
                                                         o_row_stride, do_row_stride, o_head_stride, delta, p, nullptr,
                                                         nullptr, (cudaStream_t)st);
#define FSB_BWD(DD, BB, DR)                                                                                              \
  launch_attn_bwd<DD, BB, DR>(q, k, v, o, dout, q_row_stride, k_row_stride, v_row_stride, o_row_stride, do_row_stride,       \
                          o_head_stride, delta, p, drel_bias, part2, (cudaStream_t)st)
  if (drop != nullptr) {
    p.drop = *drop;
    if (rel_bias != nullptr) return head_dim == 128 ? FSB_BWD(128, true, true) : FSB_BWD(64, true, true);
    return head_dim == 128 ? FSB_BWD(128, false, true) : FSB_BWD(64, false, true);
  }
  if (rel_bias != nullptr) return head_dim == 128 ? FSB_BWD(128, true, false) : FSB_BWD(64, true, false);
  return head_dim == 128 ? FSB_BWD(128, false, false) : FSB_BWD(64, false, false);
#undef FSB_BWD
}

extern "C" int fsb_sdpa_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout,
                            const float* lse, float* delta, void* dq, void* dk, void* dv, int64_t batch, int64_t seq_q,
                            int64_t seq_kv, int nheads, int head_dim, int64_t q_row_stride, int64_t k_row_stride,
                            int64_t v_row_stride, int64_t o_row_stride, int64_t do_row_stride, int64_t dq_row_stride,
                            int64_t dk_row_stride, int64_t dv_row_stride, int64_t q_head_stride, int64_t k_head_stride,
                            int64_t v_head_stride, int64_t o_head_stride, int64_t do_head_stride,
                            int64_t dq_head_stride, int64_t dk_head_stride, int64_t dv_head_stride, float scale,
                            int causal, const uint8_t* kv_mask, const float* rel_bias, float* drel_bias, void* workspace,
                            size_t workspace_bytes, fsb_stream_t st) {
  return sdpa_bwd(q, k, v, o, dout, lse, delta, dq, dk, dv, batch, seq_q, seq_kv, nheads, head_dim, q_row_stride,
                  k_row_stride, v_row_stride, o_row_stride, do_row_stride, dq_row_stride, dk_row_stride, dv_row_stride,
                  q_head_stride, k_head_stride, v_head_stride, o_head_stride, do_head_stride, dq_head_stride,
                  dk_head_stride, dv_head_stride, scale, causal, kv_mask, rel_bias, drel_bias, workspace, workspace_bytes,
                  nullptr, nullptr, nullptr, st);
}

extern "C" int fsb_sdpa_bwd_dropout(const void* q, const void* k, const void* v, const void* o, const void* dout,
                                    const float* lse, float* delta, void* dq, void* dk, void* dv, int64_t batch,
                                    int64_t seq_q, int64_t seq_kv, int nheads, int head_dim, int64_t q_row_stride,
                                    int64_t k_row_stride, int64_t v_row_stride, int64_t o_row_stride,
                                    int64_t do_row_stride, int64_t dq_row_stride, int64_t dk_row_stride,
                                    int64_t dv_row_stride, int64_t q_head_stride, int64_t k_head_stride,
                                    int64_t v_head_stride, int64_t o_head_stride, int64_t do_head_stride,
                                    int64_t dq_head_stride, int64_t dk_head_stride, int64_t dv_head_stride, float scale,
                                    int causal, const uint8_t* kv_mask, const float* rel_bias, float* drel_bias,
                                    void* workspace, size_t workspace_bytes, float p, uint64_t seed,
                                    const int64_t* stream_base, int64_t site, fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  // causal composes with p > 0 as in fsb_sdpa_fwd_dropout: masked elements have P = 0, so their keep bits never matter
  if (p > 0.f)
    FSB_REQUIRE(seq_q <= 65536 && seq_kv <= 65536, "sdpa_bwd_dropout: sequences longer than 65536 are not supported with p > 0");
  return sdpa_bwd(q, k, v, o, dout, lse, delta, dq, dk, dv, batch, seq_q, seq_kv, nheads, head_dim, q_row_stride,
                  k_row_stride, v_row_stride, o_row_stride, do_row_stride, dq_row_stride, dk_row_stride, dv_row_stride,
                  q_head_stride, k_head_stride, v_head_stride, o_head_stride, do_head_stride, dq_head_stride,
                  dk_head_stride, dv_head_stride, scale, causal, kv_mask, rel_bias, drel_bias, workspace, workspace_bytes,
                  p > 0.f ? &d : nullptr, nullptr, nullptr, st);
}

extern "C" int fsb_sdpa_bwd_segments(const void* q, const void* k, const void* v, const void* o, const void* dout,
                                     const float* lse, float* delta, void* dq, void* dk, void* dv, int64_t batch,
                                     int64_t seq_q, int64_t seq_kv, int nheads, int head_dim, int64_t q_row_stride,
                                     int64_t k_row_stride, int64_t v_row_stride, int64_t o_row_stride,
                                     int64_t do_row_stride, int64_t dq_row_stride, int64_t dk_row_stride,
                                     int64_t dv_row_stride, int64_t q_head_stride, int64_t k_head_stride,
                                     int64_t v_head_stride, int64_t o_head_stride, int64_t do_head_stride,
                                     int64_t dq_head_stride, int64_t dk_head_stride, int64_t dv_head_stride, float scale,
                                     const int32_t* seg_start, const int32_t* seg_end, fsb_stream_t st) {
  FSB_REQUIRE(seg_start && seg_end, "sdpa_bwd_segments: null segment bounds");
  FSB_REQUIRE(seq_q == seq_kv, "sdpa_bwd_segments: needs seq_q == seq_kv (got %lld and %lld)", (long long)seq_q,
              (long long)seq_kv);
  FSB_REQUIRE(head_dim == 64 || head_dim == 128, "sdpa_bwd_segments: head_dim %d unsupported (64 or 128)", head_dim);
  return sdpa_bwd(q, k, v, o, dout, lse, delta, dq, dk, dv, batch, seq_q, seq_kv, nheads, head_dim, q_row_stride,
                  k_row_stride, v_row_stride, o_row_stride, do_row_stride, dq_row_stride, dk_row_stride, dv_row_stride,
                  q_head_stride, k_head_stride, v_head_stride, o_head_stride, do_head_stride, dq_head_stride,
                  dk_head_stride, dv_head_stride, scale, 1, nullptr, nullptr, nullptr, nullptr, 0, nullptr, seg_start,
                  seg_end, st);
}

extern "C" int fsb_sdpa_bwd_segments_dropout(const void* q, const void* k, const void* v, const void* o, const void* dout,
                                             const float* lse, float* delta, void* dq, void* dk, void* dv, int64_t batch,
                                             int64_t seq_q, int64_t seq_kv, int nheads, int head_dim,
                                             int64_t q_row_stride, int64_t k_row_stride, int64_t v_row_stride,
                                             int64_t o_row_stride, int64_t do_row_stride, int64_t dq_row_stride,
                                             int64_t dk_row_stride, int64_t dv_row_stride, int64_t q_head_stride,
                                             int64_t k_head_stride, int64_t v_head_stride, int64_t o_head_stride,
                                             int64_t do_head_stride, int64_t dq_head_stride, int64_t dk_head_stride,
                                             int64_t dv_head_stride, float scale, const int32_t* seg_start,
                                             const int32_t* seg_end, float p, uint64_t seed, const int64_t* stream_base,
                                             int64_t site, fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  FSB_REQUIRE(seg_start && seg_end, "sdpa_bwd_segments_dropout: null segment bounds");
  FSB_REQUIRE(seq_q == seq_kv, "sdpa_bwd_segments_dropout: needs seq_q == seq_kv (got %lld and %lld)", (long long)seq_q,
              (long long)seq_kv);
  FSB_REQUIRE(head_dim == 64 || head_dim == 128, "sdpa_bwd_segments_dropout: head_dim %d unsupported (64 or 128)",
              head_dim);
  if (p > 0.f) {
    // GPT-2 (the one model with attention dropout that packs) runs head_dim 64; LLaMA has no attention dropout
    FSB_REQUIRE(head_dim == 64, "sdpa_bwd_segments_dropout: head_dim %d unsupported with p > 0 (64 only)", head_dim);
    FSB_REQUIRE(seq_q <= 65536, "sdpa_bwd_segments_dropout: sequences longer than 65536 are not supported with p > 0");
  }
  return sdpa_bwd(q, k, v, o, dout, lse, delta, dq, dk, dv, batch, seq_q, seq_kv, nheads, head_dim, q_row_stride,
                  k_row_stride, v_row_stride, o_row_stride, do_row_stride, dq_row_stride, dk_row_stride, dv_row_stride,
                  q_head_stride, k_head_stride, v_head_stride, o_head_stride, do_head_stride, dq_head_stride,
                  dk_head_stride, dv_head_stride, scale, 1, nullptr, nullptr, nullptr, nullptr, 0, p > 0.f ? &d : nullptr,
                  seg_start, seg_end, st);
}

extern "C" int fsb_sdpa_bwd_segments_bidirectional(const void* q, const void* k, const void* v, const void* o,
                                                   const void* dout, const float* lse, float* delta, void* dq, void* dk,
                                                   void* dv, int64_t batch, int64_t seq_q, int64_t seq_kv, int nheads,
                                                   int head_dim, int64_t q_row_stride, int64_t k_row_stride,
                                                   int64_t v_row_stride, int64_t o_row_stride, int64_t do_row_stride,
                                                   int64_t dq_row_stride, int64_t dk_row_stride, int64_t dv_row_stride,
                                                   int64_t q_head_stride, int64_t k_head_stride, int64_t v_head_stride,
                                                   int64_t o_head_stride, int64_t do_head_stride, int64_t dq_head_stride,
                                                   int64_t dk_head_stride, int64_t dv_head_stride, float scale,
                                                   const int32_t* seg_start, const int32_t* seg_end, float p,
                                                   uint64_t seed, const int64_t* stream_base, int64_t site,
                                                   fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  FSB_REQUIRE(seg_start && seg_end, "sdpa_bwd_segments_bidirectional: null segment bounds");
  FSB_REQUIRE(seq_q == seq_kv, "sdpa_bwd_segments_bidirectional: needs seq_q == seq_kv (got %lld and %lld)",
              (long long)seq_q, (long long)seq_kv);
  FSB_REQUIRE(head_dim == 64, "sdpa_bwd_segments_bidirectional: head_dim %d unsupported (64 only)", head_dim);
  if (p > 0.f)
    FSB_REQUIRE(seq_q <= 65536,
                "sdpa_bwd_segments_bidirectional: sequences longer than 65536 are not supported with p > 0");
  return sdpa_bwd(q, k, v, o, dout, lse, delta, dq, dk, dv, batch, seq_q, seq_kv, nheads, head_dim, q_row_stride,
                  k_row_stride, v_row_stride, o_row_stride, do_row_stride, dq_row_stride, dk_row_stride, dv_row_stride,
                  q_head_stride, k_head_stride, v_head_stride, o_head_stride, do_head_stride, dq_head_stride,
                  dk_head_stride, dv_head_stride, scale, 0, nullptr, nullptr, nullptr, nullptr, 0, p > 0.f ? &d : nullptr,
                  seg_start, seg_end, st);
}

extern "C" size_t fsb_sdpa_bwd_workspace_bytes(int64_t batch, int64_t seq_q, int64_t seq_kv, int nheads) {
  if (batch <= 0 || seq_q <= 0 || seq_kv <= 0 || nheads <= 0) return 0;
  // per-step diagonal sums of the dQ kernel + the batch-split partial vectors of the reduction
  return (fsb::dbias_part_floats(batch, seq_q, seq_kv, nheads) +
          size_t(fsb::dbias_bsplit(int(batch))) * nheads * size_t(seq_q + seq_kv - 1)) * sizeof(float);
}
