// fsb200 — KV-cache maintenance of a decode step that reads no host-side position, so that the step can be a CUDA graph.
//
//   kv_append_kernel  : copies the newest token's K and V rows (one per (row, head)) into cache slot *kv_len - 1, one 16-byte
//                       vector per thread, and optionally sets kv_mask[row, slot] = 1. Source and cache are strided views, so
//                       one entry serves the packed [t, {q,k,v}, head, d] projection of GPT-2 / mT5 with a [rows, cap, 2, heads,
//                       d] cache as well as LLaMA's interleaved [t, head, {q,k,v}, d] projection with separate K and V caches.
//   kv_reorder_kernel : the beam-search gather dst[l, r, s] = src[l, index[r], s] over the caches of every layer in one launch,
//                       restricted to the live slots s < *kv_len. CTA = (chunk of a row's live slots, row, layer).
// *kv_len is the device int32 scalar fsb_attn_decode reads; neither kernel takes a host-side position, so a captured step
// advances it on the device and replays unchanged.
#include <cuda_bf16.h>

#include "host_common.h"

namespace fsb {

constexpr int KV_THREADS = 256;
constexpr int KV_VPT = 4;   // 16-byte vectors in flight per thread in the reorder

struct AppendParams {
  const __nv_bfloat16 *k_new, *v_new;
  __nv_bfloat16 *k_cache, *v_cache;
  uint8_t* kv_mask;          // [rows, kv_cap] or nullptr
  const int32_t* kv_len;
  int64_t kn_rs, kn_hs, vn_rs, vn_hs;               // source (row, head) strides
  int64_t kc_bs, kc_ss, kc_hs, vc_bs, vc_ss, vc_hs; // cache (row, slot, head) strides
  int64_t total;             // rows * nheads * vecs
  int nheads, vecs, kv_cap;
};

__global__ void __launch_bounds__(KV_THREADS) kv_append_kernel(const AppendParams p) {
  const int64_t i = int64_t(blockIdx.x) * KV_THREADS + threadIdx.x;
  if (i >= p.total) return;
  const int slot = *p.kv_len - 1;
  if (slot < 0 || slot >= p.kv_cap) return;   // a slot outside the cache writes nothing
  const int vec = int(i % p.vecs);
  const int64_t rh = i / p.vecs;
  const int head = int(rh % p.nheads);
  const int64_t row = rh / p.nheads;
  const int64_t d = int64_t(vec) * 8;
  const uint4 k = __ldg(reinterpret_cast<const uint4*>(p.k_new + row * p.kn_rs + head * p.kn_hs + d));
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(p.v_new + row * p.vn_rs + head * p.vn_hs + d));
  *reinterpret_cast<uint4*>(p.k_cache + row * p.kc_bs + slot * p.kc_ss + head * p.kc_hs + d) = k;
  *reinterpret_cast<uint4*>(p.v_cache + row * p.vc_bs + slot * p.vc_ss + head * p.vc_hs + d) = v;
  if (p.kv_mask != nullptr && head == 0 && vec == 0) p.kv_mask[row * p.kv_cap + slot] = 1;
}

struct ReorderParams {
  const uint4* src;
  uint4* dst;
  const int64_t* index;      // [rows]
  const int32_t* kv_len;
  int64_t rows, kv_cap, slot_vecs;
};

__global__ void __launch_bounds__(KV_THREADS) kv_reorder_kernel(const ReorderParams p) {
  const int64_t row = blockIdx.y, layer = blockIdx.z;
  int64_t n = *p.kv_len;
  n = n < 0 ? 0 : (n > p.kv_cap ? p.kv_cap : n);
  const int64_t live = n * p.slot_vecs;
  const int64_t c0 = int64_t(blockIdx.x) * (KV_THREADS * KV_VPT);
  if (c0 >= live) return;                     // this chunk holds no live slot: read and write nothing
  const int64_t from = p.index[row];
  if (from < 0 || from >= p.rows) return;     // an out-of-range source row leaves the destination row untouched
  const uint4* s = p.src + (layer * p.rows + from) * p.kv_cap * p.slot_vecs;
  uint4* d = p.dst + (layer * p.rows + row) * p.kv_cap * p.slot_vecs;
  uint4 r[KV_VPT];
#pragma unroll
  for (int u = 0; u < KV_VPT; ++u) {
    const int64_t j = c0 + u * KV_THREADS + threadIdx.x;
    if (j < live) r[u] = __ldg(s + j);
  }
#pragma unroll
  for (int u = 0; u < KV_VPT; ++u) {
    const int64_t j = c0 + u * KV_THREADS + threadIdx.x;
    if (j < live) d[j] = r[u];
  }
}

}  // namespace fsb

using namespace fsb;

extern "C" int fsb_kv_append(const void* k_new, const void* v_new, void* k_cache, void* v_cache, uint8_t* kv_mask,
                             int64_t rows, int nheads, int head_dim, int64_t kv_cap, const int32_t* kv_len,
                             int64_t k_new_row_stride, int64_t k_new_head_stride, int64_t v_new_row_stride,
                             int64_t v_new_head_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t k_head_stride,
                             int64_t v_batch_stride, int64_t v_row_stride, int64_t v_head_stride, fsb_stream_t st) {
  FSB_REQUIRE(k_new && v_new && k_cache && v_cache && kv_len, "kv_append: null pointer");
  FSB_REQUIRE(rows > 0 && nheads > 0 && kv_cap > 0 && kv_cap < (int64_t(1) << 30) && head_dim > 0 && head_dim % 8 == 0,
              "kv_append: bad dims (rows %lld, nheads %d, head_dim %d, kv_cap %lld)", (long long)rows, nheads, head_dim,
              (long long)kv_cap);
  FSB_REQUIRE(aligned16(k_new) && aligned16(v_new) && aligned16(k_cache) && aligned16(v_cache),
              "kv_append: 16-byte alignment required");
  FSB_REQUIRE((k_new_row_stride | k_new_head_stride | v_new_row_stride | v_new_head_stride | k_batch_stride | k_row_stride |
               k_head_stride | v_batch_stride | v_row_stride | v_head_stride) % 8 == 0,
              "kv_append: strides must be multiples of 8 elements");
  AppendParams p;
  p.k_new = (const __nv_bfloat16*)k_new; p.v_new = (const __nv_bfloat16*)v_new;
  p.k_cache = (__nv_bfloat16*)k_cache; p.v_cache = (__nv_bfloat16*)v_cache;
  p.kv_mask = kv_mask; p.kv_len = kv_len;
  p.kn_rs = k_new_row_stride; p.kn_hs = k_new_head_stride; p.vn_rs = v_new_row_stride; p.vn_hs = v_new_head_stride;
  p.kc_bs = k_batch_stride; p.kc_ss = k_row_stride; p.kc_hs = k_head_stride;
  p.vc_bs = v_batch_stride; p.vc_ss = v_row_stride; p.vc_hs = v_head_stride;
  p.nheads = nheads; p.vecs = head_dim / 8; p.kv_cap = int(kv_cap);
  p.total = rows * nheads * p.vecs;
  const int64_t blocks = (p.total + KV_THREADS - 1) / KV_THREADS;
  FSB_REQUIRE(blocks < (int64_t(1) << 31), "kv_append: too many rows");
  kv_append_kernel<<<unsigned(blocks), KV_THREADS, 0, (cudaStream_t)st>>>(p);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

extern "C" int fsb_kv_reorder(const void* src, void* dst, const int64_t* index, int64_t layers, int64_t rows, int64_t kv_cap,
                              int64_t slot_elems, const int32_t* kv_len, fsb_stream_t st) {
  FSB_REQUIRE(src && dst && index && kv_len, "kv_reorder: null pointer");
  FSB_REQUIRE(layers > 0 && layers < 65536 && rows > 0 && rows < 65536 && kv_cap > 0 && kv_cap < (int64_t(1) << 30) &&
                  slot_elems > 0 && slot_elems % 8 == 0,
              "kv_reorder: bad dims (layers %lld, rows %lld, kv_cap %lld, slot_elems %lld)", (long long)layers,
              (long long)rows, (long long)kv_cap, (long long)slot_elems);
  FSB_REQUIRE(aligned16(src) && aligned16(dst), "kv_reorder: 16-byte alignment required");
  const uintptr_t bytes = uintptr_t(layers) * rows * kv_cap * slot_elems * 2;
  const uintptr_t s = reinterpret_cast<uintptr_t>(src), d = reinterpret_cast<uintptr_t>(dst);
  FSB_REQUIRE(s + bytes <= d || d + bytes <= s, "kv_reorder: source and destination caches overlap");
  ReorderParams p;
  p.src = static_cast<const uint4*>(src); p.dst = static_cast<uint4*>(dst); p.index = index; p.kv_len = kv_len;
  p.rows = rows; p.kv_cap = kv_cap; p.slot_vecs = slot_elems / 8;
  const int64_t chunks = (kv_cap * p.slot_vecs + KV_THREADS * KV_VPT - 1) / (KV_THREADS * KV_VPT);
  FSB_REQUIRE(chunks < (int64_t(1) << 31), "kv_reorder: cache rows too long");
  kv_reorder_kernel<<<dim3(unsigned(chunks), unsigned(rows), unsigned(layers)), KV_THREADS, 0, (cudaStream_t)st>>>(p);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
