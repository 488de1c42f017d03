// fsb200 — fused scaled-dot-product attention, forward (flash-style online softmax on wgmma).
// Replaces ParallelSelfAttention.flash_attention (fengshen/models/megatron/layers/transformer.py:410-456, 3P
// flash_attn_cuda.fwd) and the baddbmm -> FusedScaleMaskSoftmax -> bmm path (transformer.py:307-408): same math,
//   O = softmax(scale * Q K^T + mask) V,  mask = causal and/or key-padding,
// without the three repacking copies of q/k/v (transformer.py:419-429): Q, K, V are read straight out of the packed
// QKV projection output through TMA tensor maps (any row/head stride), O is written in [token, head*dim] layout.
//
// CTA = one (batch, head, 128-row Q tile), 3 warpgroups:
//   warpgroup 0     : TMA producer (Q once; K and V tiles through a multi-stage ring, separate full barriers so that
//                     S = Q K^T can start before V has landed)
//   warpgroups 1, 2 : 64 query rows each. S(j) = Q K_j^T (wgmma, both operands in shared memory, fp32 in registers),
//                     online softmax in registers (a row lives in the four lanes of a quad), then O += P(j) V_j with P as
//                     the register A operand — P never touches shared memory.
// The two consumer warpgroups run independently on the same K/V stage, so one's softmax overlaps the other's MMAs.
#include <stdlib.h>

#include "host_common.h"
#include "ptx.cuh"

namespace fsb {

constexpr int ATT_BQ = 128;   // rows per Q tile (two consumer warpgroups x 64)
constexpr int ATT_BKV = 128;  // keys per inner step
constexpr int ATT_THREADS = 384;

template <int D>
struct AttFwdSmem {
  static constexpr int STAGES = D == 128 ? 2 : 3;          // K/V ring depth
  static constexpr int Q_BYTES = ATT_BQ * D * 2;
  static constexpr int KV_BYTES = ATT_BKV * D * 2;         // per tensor per stage
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + Q_BYTES;
  static constexpr int OFF_V = OFF_K + STAGES * KV_BYTES;
  static constexpr int OFF_BAR = OFF_V + STAGES * KV_BYTES;
  // q_full, k_full[S], v_full[S], kv_empty[S]
  static constexpr int NBAR = 1 + 3 * STAGES;
  static constexpr int TOTAL = OFF_BAR + NBAR * 8 + 1024;
  static_assert(TOTAL <= 232448, "exceeds the 227 KB of shared memory a block can opt into on sm_90");
};

struct AttFwdParams {
  __nv_bfloat16* o;
  float* lse;               // [batch, nheads, seq_q], log2 domain
  const uint8_t* kv_mask;   // [batch, seq_kv] (1 = attend) or nullptr
  const float* rel_bias;    // [nheads, seq_q + seq_kv - 1] additive bias over the offset k - q (natural-log units) or nullptr
  int64_t o_row_stride, o_head_stride;
  int q_head_stride, k_head_stride, v_head_stride;
  int seq_q, seq_kv, nheads, batch;
  int causal;
  float scale_log2;  // softmax scale * log2(e)
};

template <int D>
__device__ __forceinline__ void wgmma_rs_d(float (&o)[D / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (D == 128) wgmma_rs_n128<1>(o, a, db, 1u);
  else wgmma_rs_n64<1>(o, a, db, 1u);
}

template <int D, bool kBias>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttFwdParams p) {
  using S = AttFwdSmem<D>;
  constexpr int STAGES = S::STAGES;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* k_full = q_full + 1;
  uint64_t* v_full = k_full + STAGES;
  uint64_t* kv_empty = v_full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = gridDim.x - 1 - blockIdx.x;  // heavy (late) causal tiles first
  const int head = blockIdx.y, b = blockIdx.z;
  const int q0 = tile * ATT_BQ;
  const int n_all = (p.seq_kv + ATT_BKV - 1) / ATT_BKV;
  const int n_kv = p.causal ? min(n_all, (min(q0 + ATT_BQ, p.seq_q) + ATT_BKV - 1) / ATT_BKV) : n_all;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&k_full[i], 1); mbar_init(&v_full[i], 1);
      mbar_init(&kv_empty[i], 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    reg_dec<24>();
    if (threadIdx.x == 0) {
      const int qc = head * p.q_head_stride, kc = head * p.k_head_stride, vc = head * p.v_head_stride;
      mbar_expect_tx(q_full, S::Q_BYTES);
#pragma unroll
      for (int h = 0; h < D / 64; ++h) tma_load_3d(smem + S::OFF_Q + h * (ATT_BQ * 128), &tmQ, q_full, qc + h * 64, q0, b);
      int st = 0; uint32_t ph = 0;
      for (int j = 0; j < n_kv; ++j) {
        mbar_wait(&kv_empty[st], ph ^ 1);
        mbar_expect_tx(&k_full[st], S::KV_BYTES);
#pragma unroll
        for (int h = 0; h < D / 64; ++h)
          tma_load_3d(smem + S::OFF_K + st * S::KV_BYTES + h * (ATT_BKV * 128), &tmK, &k_full[st], kc + h * 64, j * ATT_BKV, b);
        mbar_expect_tx(&v_full[st], S::KV_BYTES);
#pragma unroll
        for (int h = 0; h < D / 64; ++h)
          tma_load_3d(smem + S::OFF_V + st * S::KV_BYTES + h * (ATT_BKV * 128), &tmV, &v_full[st], vc + h * 64, j * ATT_BKV, b);
        if (++st == STAGES) { st = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile =====================
  reg_inc<240>();   // 256 * 240 + 128 * 24 = 64512
  const int wg = (threadIdx.x >> 7) - 1;
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: r_lo and r_lo + 8
  const int cq = 2 * (lane & 3);                               // its columns inside every 8-column group: cq, cq + 1
  const uint64_t dsc_q = make_smem_desc_sw128(smem_u32(smem + S::OFF_Q) + wg * (64 * 128), 0, 1024);
  const uint64_t dsc_k = make_smem_desc_sw128(smem_u32(smem + S::OFF_K), 0, 1024);
  const uint64_t dsc_v = make_smem_desc_sw128(smem_u32(smem + S::OFF_V), ATT_BKV * 128, 1024);   // MN-major (D contiguous)
  const uint8_t* mrow = p.kv_mask ? p.kv_mask + int64_t(b) * p.seq_kv : nullptr;
  const float sc = p.scale_log2;
  const int n_rel = p.seq_q + p.seq_kv - 1;
  int q_row[2], kmax[2];
  const float* brow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    q_row[h] = q0 + r_lo + 8 * h;
    kmax[h] = p.causal ? min(q_row[h], p.seq_kv - 1) : p.seq_kv - 1;   // last key column this row may attend to
    // T5 / mT5 relative-position bias (transformers mt5/modeling_mt5.py:181-235,:320): bias[h, q, k] depends on k - q only, so
    // it arrives as one vector per head; this row reads entries (k - q_row + seq_q - 1).
    brow[h] = kBias ? p.rel_bias + int64_t(head) * n_rel + (p.seq_q - 1 - min(q_row[h], p.seq_q - 1)) : nullptr;
  }
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // running max (scaled log2 domain), thread-partial row sums

  mbar_wait(q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int st = j % STAGES;
    const uint32_t ph = (j / STAGES) & 1;
    float s[ATT_BKV / 2];
    mbar_wait(&k_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_ss_n128<0, 0>(s, dsc_q + (((kk / 4) * (ATT_BQ * 128) + (kk % 4) * 32) >> 4),
                          dsc_k + ((st * S::KV_BYTES + (kk / 4) * (ATT_BKV * 128) + (kk % 4) * 32) >> 4), kk != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);

    // scores -> scaled log2 domain (+ bias), masked to -inf; s[4 i + e]: column 8 i + cq + (e & 1), row h = e >> 1
    const int c0 = j * ATT_BKV;
    const bool need_mask = (p.causal && c0 + ATT_BKV - 1 > q0 + wg * 64) || (c0 + ATT_BKV > p.seq_kv) || mrow;
#pragma unroll
    for (int i = 0; i < ATT_BKV / 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int h = e >> 1, col = c0 + 8 * i + cq + (e & 1);
        float x;
        if constexpr (kBias) x = fmaf(__ldg(brow[h] + min(col, p.seq_kv - 1)), 1.4426950408889634f, s[4 * i + e] * sc);
        else x = s[4 * i + e] * sc;
        if (need_mask) {
          bool keep = col <= kmax[h];
          if (mrow != nullptr && keep) keep = mrow[col] != 0;
          x = keep ? x : -INFINITY;
        }
        s[4 * i + e] = x;
      }
    }
    float neg_m[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < ATT_BKV / 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * h], s[4 * i + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx);
      const float f = (m_new == -INFINITY) ? 1.f : ex2_approx(m[h] - m_new);
      l[h] *= f;
#pragma unroll
      for (int i = 0; i < D / 8; ++i) { o[4 * i + 2 * h] *= f; o[4 * i + 2 * h + 1] *= f; }
      m[h] = m_new;
      neg_m[h] = (m_new == -INFINITY) ? 0.f : -m_new;
    }
    // P(j) as register A fragments: 16-key slice kk = accumulator groups 2 kk and 2 kk + 1
    uint32_t pa[ATT_BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < ATT_BKV / 16; ++kk) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int h = r & 1, i = 2 * kk + (r >> 1);
        const float a = ex2_approx(s[4 * i + 2 * h] + neg_m[h]), c = ex2_approx(s[4 * i + 2 * h + 1] + neg_m[h]);
        l[h] += a + c;   // fp32 sums of the unrounded probabilities
        pa[kk][r] = pack_bf16x2(a, c);
      }
    }
    mbar_wait(&v_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BKV / 16; ++kk)
      wgmma_rs_d<D>(o, pa[kk], dsc_v + ((st * S::KV_BYTES + kk * 2048) >> 4));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
  }

  // ---- epilogue: normalise, store O (bf16) and LSE (log2 domain)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float lr = l[h];
    lr += __shfl_xor_sync(0xffffffffu, lr, 1);
    lr += __shfl_xor_sync(0xffffffffu, lr, 2);
    if (q_row[h] >= p.seq_q) continue;
    const float inv = lr > 0.f ? 1.f / lr : 0.f;
    __nv_bfloat16* op = p.o + (int64_t(b) * p.seq_q + q_row[h]) * p.o_row_stride + int64_t(head) * p.o_head_stride + cq;
#pragma unroll
    for (int i = 0; i < D / 8; ++i)
      *reinterpret_cast<uint32_t*>(op + 8 * i) = pack_bf16x2(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
    if ((lane & 3) == 0)
      p.lse[(int64_t(b) * p.nheads + head) * p.seq_q + q_row[h]] = lr > 0.f ? m[h] + log2f(lr) : INFINITY;
  }
}

// Tensor map over a packed activation buffer: dims {row_width, seq, batch}; box {64, box_rows, 1}.
int make_attn_tmap(CUtensorMap* tm, const void* base, int64_t row_stride, int64_t width, int64_t seq, int64_t batch,
                   int box_rows) {
  uint64_t dims[3] = {uint64_t(width), uint64_t(seq), uint64_t(batch)};
  uint64_t strides[2] = {uint64_t(row_stride) * 2, uint64_t(seq) * uint64_t(row_stride) * 2};
  uint32_t box[3] = {64, uint32_t(box_rows), 1};
  return make_tmap_bf16(tm, base, 3, dims, strides, box);
}

template <int D, bool kBias>
static int launch_attn_fwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttFwdParams& p,
                           cudaStream_t st) {
  using S = AttFwdSmem<D>;
  static bool configured = false;
  auto kern = attn_fwd_kernel<D, kBias>;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL);
    if (e != cudaSuccess) {
      set_error("sdpa_fwd: cudaFuncSetAttribute(%d) failed: %s", S::TOTAL, cudaGetErrorString(e));
      return FSB_ERR_CUDA;
    }
    configured = true;
  }
  dim3 grid((p.seq_q + ATT_BQ - 1) / ATT_BQ, p.nheads, p.batch);
  kern<<<grid, ATT_THREADS, S::TOTAL, st>>>(tq, tk, tv, p);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

}  // namespace fsb

using namespace fsb;

extern "C" int fsb_sdpa_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int64_t batch,
                            int64_t seq_q, int64_t seq_kv, int nheads, int head_dim, int64_t q_row_stride,
                            int64_t k_row_stride, int64_t v_row_stride, int64_t o_row_stride, int64_t q_head_stride,
                            int64_t k_head_stride, int64_t v_head_stride, int64_t o_head_stride, float scale, int causal,
                            const uint8_t* kv_mask, const float* rel_bias, fsb_stream_t st) {
  FSB_REQUIRE(q && k && v && o && lse, "sdpa_fwd: null pointer");
  FSB_REQUIRE(head_dim == 64 || head_dim == 128, "sdpa_fwd: head_dim %d unsupported (64 or 128)", head_dim);
  FSB_REQUIRE(batch > 0 && seq_q > 0 && seq_kv > 0 && nheads > 0 && batch < 65536 && nheads < 65536, "sdpa_fwd: bad dims");
  FSB_REQUIRE(!causal || seq_q == seq_kv, "sdpa_fwd: causal needs seq_q == seq_kv");
  FSB_REQUIRE(scale > 0.f, "sdpa_fwd: softmax scale must be positive");
  FSB_REQUIRE(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(o), "sdpa_fwd: 16-byte alignment required");
  FSB_REQUIRE((q_row_stride | k_row_stride | v_row_stride | o_row_stride | q_head_stride | k_head_stride |
               v_head_stride | o_head_stride) % 8 == 0,
              "sdpa_fwd: strides must be multiples of 8 elements");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_attn_tmap(&tq, q, q_row_stride, (nheads - 1) * q_head_stride + head_dim, seq_q, batch, ATT_BQ))) return rc;
  if ((rc = make_attn_tmap(&tk, k, k_row_stride, (nheads - 1) * k_head_stride + head_dim, seq_kv, batch, ATT_BKV))) return rc;
  if ((rc = make_attn_tmap(&tv, v, v_row_stride, (nheads - 1) * v_head_stride + head_dim, seq_kv, batch, ATT_BKV))) return rc;
  AttFwdParams p;
  p.o = (__nv_bfloat16*)o; p.lse = lse; p.kv_mask = kv_mask; p.rel_bias = rel_bias;
  p.o_row_stride = o_row_stride; p.o_head_stride = o_head_stride;
  p.q_head_stride = int(q_head_stride); p.k_head_stride = int(k_head_stride); p.v_head_stride = int(v_head_stride);
  p.seq_q = int(seq_q); p.seq_kv = int(seq_kv); p.nheads = nheads; p.batch = int(batch);
  p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  if (rel_bias != nullptr)
    return head_dim == 128 ? launch_attn_fwd<128, true>(tq, tk, tv, p, (cudaStream_t)st)
                           : launch_attn_fwd<64, true>(tq, tk, tv, p, (cudaStream_t)st);
  return head_dim == 128 ? launch_attn_fwd<128, false>(tq, tk, tv, p, (cudaStream_t)st)
                         : launch_attn_fwd<64, false>(tq, tk, tv, p, (cudaStream_t)st);
}
