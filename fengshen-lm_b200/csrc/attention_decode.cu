// fsb200 — decode attention: one query row per (batch, head) against a pre-allocated KV cache, split over the keys.
//
// A decode step of an autoregressive model (GPT-2, the mT5 decoder) attends from the newest token, which sits at cache slot
// *kv_len - 1, to the slots [0, *kv_len). The work per (batch, head) is one HBM pass over 2 * kv_len * head_dim bf16 values and
// almost no arithmetic, and batch * heads is often below the SM count, so the keys are split into chunks and every chunk is a
// CTA of its own (split-KV, as in FlashDecoding):
//   attn_decode_kernel  : CTA = (chunk, head, batch), 4 warps. head_dim / 8 lanes own one key (16-byte vector loads of K and
//                         V, 8 elements a lane), so a warp holds 32 / (head_dim / 8) keys at a time and every lane keeps an
//                         fp32 online softmax (m, l, acc[8]) over the keys its lane group visits. The lane groups and then the
//                         warps are merged in a fixed order, and the CTA writes one fp32 partial (m, l, acc[head_dim]).
//                         A CTA whose chunk starts at or beyond *kv_len writes an empty partial (l = 0) and reads nothing,
//                         so HBM traffic follows kv_len, not kv_cap.
//   attn_decode_combine : CTA = (head, batch); merges the partials in split order and writes O (bf16) and the LSE.
// The split plan depends only on (batch, nheads, kv_cap), never on *kv_len, so *kv_len can live on the device (a graph-captured
// decode loop can advance it without re-planning) and two identical calls produce identical bits.
#include <math.h>

#include "host_common.h"
#include "ptx.cuh"

namespace fsb {

constexpr int DEC_THREADS = 128;
constexpr int DEC_WARPS = DEC_THREADS / 32;
constexpr int DEC_UNROLL = 4;       // keys in flight per lane group before the first one is consumed
constexpr int DEC_MIN_CHUNK = 64;   // keys per split at least: below that the merge costs more than the keys
constexpr int DEC_CTAS_PER_SM = 4;  // 4 x 128 threads x 8 x 16 B in flight per SM covers the HBM latency

struct DecodeParams {
  const __nv_bfloat16 *q, *k, *v;
  __nv_bfloat16* o;
  float* lse;                  // [batch, nheads], log2 domain, or nullptr
  const int32_t* kv_len;       // device scalar
  const uint8_t* kv_mask;      // [batch, kv_cap] (1 = attend) or nullptr
  const float* rel_bias;       // [nheads, 2 kv_cap - 1] or nullptr
  float* part_ml;              // [batch, nheads, splits, 2]: running max (scaled log2 domain), sum of exponentials
  float* part_acc;             // [batch, nheads, splits, D]: un-normalised output
  int64_t q_bs, q_hs, k_bs, k_rs, k_hs, v_bs, v_rs, v_hs, o_bs, o_hs;
  int nheads, kv_cap, splits, chunk;
  float scale_log2;            // softmax scale * log2(e)
};

struct DecodePlan {
  int splits, chunk;
};

static DecodePlan decode_plan(int64_t batch, int nheads, int64_t kv_cap) {
  const int64_t rows = batch * nheads;
  int64_t want = (int64_t(DEC_CTAS_PER_SM) * num_sms() + rows - 1) / rows;
  const int64_t most = (kv_cap + DEC_MIN_CHUNK - 1) / DEC_MIN_CHUNK;
  if (want > most) want = most;
  if (want < 1) want = 1;
  int64_t chunk = (kv_cap + want - 1) / want;
  chunk = (chunk + DEC_MIN_CHUNK - 1) / DEC_MIN_CHUNK * DEC_MIN_CHUNK;
  return DecodePlan{int((kv_cap + chunk - 1) / chunk), int(chunk)};
}

static size_t decode_ws_bytes(int64_t batch, int nheads, int head_dim, const DecodePlan& pl) {
  return size_t(batch) * nheads * pl.splits * (head_dim + 2) * sizeof(float);
}

__device__ __forceinline__ int decode_len(const DecodeParams& p) {
  const int n = *p.kv_len;
  return n < 0 ? 0 : (n > p.kv_cap ? p.kv_cap : n);
}

// (m, l, a) <- merge of (m, l, a) and (m2, l2, a2); an empty side (m = -inf) contributes nothing.
__device__ __forceinline__ void merge_state(float& m, float& l, float (&a)[8], float m2, float l2, const float (&a2)[8]) {
  const float mx = fmaxf(m, m2);
  const float f1 = m == -INFINITY ? 0.f : ex2_approx(m - mx);
  const float f2 = m2 == -INFINITY ? 0.f : ex2_approx(m2 - mx);
  m = mx;
  l = l * f1 + l2 * f2;
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = a[i] * f1 + a2[i] * f2;
}

template <int D>
__global__ void __launch_bounds__(DEC_THREADS) attn_decode_kernel(const DecodeParams p) {
  constexpr int G = D / 8;              // lanes per key
  constexpr int KPW = 32 / G;           // keys per warp step
  constexpr int KPC = KPW * DEC_WARPS;  // keys per CTA step
  __shared__ float sm_ml[DEC_WARPS][2];
  __shared__ __align__(16) float sm_acc[DEC_WARPS][D];

  const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, grp = lane / G, sub = lane % G;
  const int64_t row = (int64_t(b) * p.nheads + head) * p.splits + split;
  const int len = decode_len(p);
  const int c0 = split * p.chunk;
  const int c1 = min(c0 + p.chunk, len);
  if (c0 >= len) {   // nothing of this chunk is in the cache yet
    if (threadIdx.x == 0) { p.part_ml[2 * row] = -INFINITY; p.part_ml[2 * row + 1] = 0.f; }
    return;
  }

  float qf[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(p.q + b * p.q_bs + head * p.q_hs) + sub), qf);
#pragma unroll
  for (int i = 0; i < 8; ++i) qf[i] *= p.scale_log2;
  const __nv_bfloat16* kb = p.k + b * p.k_bs + head * p.k_hs + sub * 8;
  const __nv_bfloat16* vb = p.v + b * p.v_bs + head * p.v_hs + sub * 8;
  const uint8_t* mrow = p.kv_mask ? p.kv_mask + int64_t(b) * p.kv_cap : nullptr;
  // bias of key k for the query at slot len - 1: rel_bias[head][k - (len - 1) + kv_cap - 1]
  const float* brow = p.rel_bias ? p.rel_bias + int64_t(head) * (2 * p.kv_cap - 1) + (p.kv_cap - len) : nullptr;

  float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;

  // the trip count is warp-uniform (shuffles below need every lane); keys past c1 are loaded as nothing and scored -inf
  for (int base = c0 + warp * KPW + grp; base - grp < c1; base += KPC * DEC_UNROLL) {
    uint4 kr[DEC_UNROLL], vr[DEC_UNROLL];
#pragma unroll
    for (int u = 0; u < DEC_UNROLL; ++u) {
      const int key = base + u * KPC;
      if (key < c1) {
        kr[u] = __ldg(reinterpret_cast<const uint4*>(kb + key * p.k_rs));
        vr[u] = __ldg(reinterpret_cast<const uint4*>(vb + key * p.v_rs));
      } else {
        kr[u] = make_uint4(0, 0, 0, 0); vr[u] = make_uint4(0, 0, 0, 0);
      }
    }
    float s[DEC_UNROLL];
#pragma unroll
    for (int u = 0; u < DEC_UNROLL; ++u) {
      float kf[8];
      unpack8(kr[u], kf);
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) d = fmaf(qf[i], kf[i], d);
#pragma unroll
      for (int off = 1; off < G; off <<= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
      const int key = base + u * KPC;
      bool keep = key < c1;
      if (keep && mrow != nullptr) keep = mrow[key] != 0;
      if (brow != nullptr && keep) d = fmaf(__ldg(brow + key), 1.4426950408889634f, d);
      s[u] = keep ? d : -INFINITY;
    }
    float mx = m;
#pragma unroll
    for (int u = 0; u < DEC_UNROLL; ++u) mx = fmaxf(mx, s[u]);
    if (mx == -INFINITY) continue;   // every key so far masked: the state stays empty
    const float f = m == -INFINITY ? 0.f : ex2_approx(m - mx);
    l *= f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] *= f;
#pragma unroll
    for (int u = 0; u < DEC_UNROLL; ++u) {
      const float pr = s[u] == -INFINITY ? 0.f : ex2_approx(s[u] - mx);
      l += pr;
      float vf[8];
      unpack8(vr[u], vf);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(pr, vf[i], acc[i]);
    }
    m = mx;
  }

  // lane groups of a warp: butterfly over the group index (a fixed tree, hence deterministic)
#pragma unroll
  for (int off = G; off < 32; off <<= 1) {
    float a2[8];
    const float m2 = __shfl_xor_sync(0xffffffffu, m, off), l2 = __shfl_xor_sync(0xffffffffu, l, off);
#pragma unroll
    for (int i = 0; i < 8; ++i) a2[i] = __shfl_xor_sync(0xffffffffu, acc[i], off);
    merge_state(m, l, acc, m2, l2, a2);
  }
  if (grp == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) sm_acc[warp][sub * 8 + i] = acc[i];
    if (sub == 0) { sm_ml[warp][0] = m; sm_ml[warp][1] = l; }
  }
  __syncthreads();
  // warps in index order; thread t < D owns output column t
  if (threadIdx.x < D) {
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < DEC_WARPS; ++w) M = fmaxf(M, sm_ml[w][0]);
    float Lsum = 0.f, A = 0.f;
#pragma unroll
    for (int w = 0; w < DEC_WARPS; ++w) {
      const float mw = sm_ml[w][0];
      const float f = mw == -INFINITY ? 0.f : ex2_approx(mw - M);
      Lsum = fmaf(sm_ml[w][1], f, Lsum);
      A = fmaf(sm_acc[w][threadIdx.x], f, A);
    }
    p.part_acc[row * D + threadIdx.x] = A;
    if (threadIdx.x == 0) { p.part_ml[2 * row] = M; p.part_ml[2 * row + 1] = Lsum; }
  }
}

template <int D>
__global__ void __launch_bounds__(D) attn_decode_combine(const DecodeParams p) {
  const int head = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const int64_t row0 = (int64_t(b) * p.nheads + head) * p.splits;
  const float* ml = p.part_ml + 2 * row0;
  float M = -INFINITY;
  for (int s = 0; s < p.splits; ++s)
    if (ml[2 * s + 1] > 0.f) M = fmaxf(M, ml[2 * s]);
  float Lsum = 0.f, A = 0.f;
  for (int s = 0; s < p.splits; ++s) {   // split order: fixed, so the result does not depend on the launch schedule
    const float ls = ml[2 * s + 1];
    if (ls > 0.f) {                        // empty partials carry no acc (it was never written)
      const float f = ex2_approx(ml[2 * s] - M);
      Lsum = fmaf(ls, f, Lsum);
      A = fmaf(p.part_acc[(row0 + s) * D + t], f, A);
    }
  }
  p.o[b * p.o_bs + head * p.o_hs + t] = __float2bfloat16(Lsum > 0.f ? A / Lsum : 0.f);
  if (t == 0 && p.lse != nullptr) p.lse[int64_t(b) * p.nheads + head] = Lsum > 0.f ? M + log2f(Lsum) : INFINITY;
}

template <int D>
static int launch_decode(const DecodeParams& p, int batch, cudaStream_t st) {
  attn_decode_kernel<D><<<dim3(p.splits, p.nheads, batch), DEC_THREADS, 0, st>>>(p);
  FSB_CUDA_LAUNCH_CHECK();
  attn_decode_combine<D><<<dim3(p.nheads, batch), D, 0, st>>>(p);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

}  // namespace fsb

using namespace fsb;

extern "C" size_t fsb_attn_decode_workspace_bytes(int64_t batch, int nheads, int head_dim, int64_t kv_cap) {
  if (batch <= 0 || nheads <= 0 || kv_cap <= 0 || (head_dim != 64 && head_dim != 128)) return 0;
  return decode_ws_bytes(batch, nheads, head_dim, decode_plan(batch, nheads, kv_cap));
}

extern "C" int fsb_attn_decode(const void* q, const void* k, const void* v, void* o, float* lse, int64_t batch, int nheads,
                               int head_dim, int64_t kv_cap, const int32_t* kv_len, int64_t q_batch_stride,
                               int64_t q_head_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t k_head_stride,
                               int64_t v_batch_stride, int64_t v_row_stride, int64_t v_head_stride, int64_t o_batch_stride,
                               int64_t o_head_stride, float scale, const uint8_t* kv_mask, const float* rel_bias,
                               void* workspace, size_t workspace_bytes, fsb_stream_t st) {
  FSB_REQUIRE(q && k && v && o && kv_len, "attn_decode: null pointer");
  FSB_REQUIRE(head_dim == 64 || head_dim == 128, "attn_decode: head_dim %d unsupported (64 or 128)", head_dim);
  FSB_REQUIRE(batch > 0 && nheads > 0 && kv_cap > 0 && batch < 65536 && nheads < 65536 && kv_cap < (int64_t(1) << 30),
              "attn_decode: bad dims (batch %lld, nheads %d, kv_cap %lld)", (long long)batch, nheads, (long long)kv_cap);
  FSB_REQUIRE(scale > 0.f, "attn_decode: softmax scale must be positive");
  FSB_REQUIRE(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(o), "attn_decode: 16-byte alignment required");
  FSB_REQUIRE((q_batch_stride | q_head_stride | k_batch_stride | k_row_stride | k_head_stride | v_batch_stride |
               v_row_stride | v_head_stride | o_batch_stride | o_head_stride) % 8 == 0,
              "attn_decode: strides must be multiples of 8 elements");
  const DecodePlan pl = decode_plan(batch, nheads, kv_cap);
  const size_t need = decode_ws_bytes(batch, nheads, head_dim, pl);
  FSB_REQUIRE(workspace != nullptr && workspace_bytes >= need && aligned16(workspace),
              "attn_decode: needs a 16-byte aligned %zu-byte workspace (fsb_attn_decode_workspace_bytes); got %zu", need,
              workspace_bytes);
  DecodeParams p;
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v;
  p.o = (__nv_bfloat16*)o; p.lse = lse; p.kv_len = kv_len; p.kv_mask = kv_mask; p.rel_bias = rel_bias;
  const int64_t rows = batch * nheads * pl.splits;
  p.part_ml = static_cast<float*>(workspace);
  p.part_acc = p.part_ml + 2 * rows;
  p.q_bs = q_batch_stride; p.q_hs = q_head_stride;
  p.k_bs = k_batch_stride; p.k_rs = k_row_stride; p.k_hs = k_head_stride;
  p.v_bs = v_batch_stride; p.v_rs = v_row_stride; p.v_hs = v_head_stride;
  p.o_bs = o_batch_stride; p.o_hs = o_head_stride;
  p.nheads = nheads; p.kv_cap = int(kv_cap); p.splits = pl.splits; p.chunk = pl.chunk;
  p.scale_log2 = scale * 1.4426950408889634f;
  return head_dim == 128 ? launch_decode<128>(p, int(batch), (cudaStream_t)st)
                         : launch_decode<64>(p, int(batch), (cudaStream_t)st);
}
