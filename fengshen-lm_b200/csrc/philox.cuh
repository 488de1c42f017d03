// fsb200 — counter-based dropout masks: Philox4x32-10 (Salmon et al., SC'11; the Random123 definition) and the counter
// layouts of include/fsb200.h. The keep bit of an element is a pure function of (seed, stream, coordinates), so any kernel —
// whatever tile, CTA or thread computes the element — can regenerate it, and no mask is ever stored.
#pragma once
#include <stdint.h>

#include "host_common.h"

namespace fsb {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

// What every dropout kernel needs: the key, the stream of its site and the 8-bit threshold. The stream is read from the
// device (base + site) so that a replayed CUDA graph draws fresh masks.
struct DropArgs {
  uint64_t seed;
  const int64_t* stream_base;   // device; the forward's base, saved with the activations
  int64_t site;
  uint32_t thr;                 // drop when the byte < thr; thr = round(p * 256)
  float keep_scale;             // 1 / (1 - p)
};

// Host side of every *_dropout entry point: validates p and fills the launch arguments. p == 0 selects the kernels without
// dropout (the callers pass nullptr instead of the arguments).
static inline int make_drop_args(float p, uint64_t seed, const int64_t* stream_base, int64_t site, DropArgs* d) {
  FSB_REQUIRE(p >= 0.f && p < 1.f, "dropout: p = %g outside [0, 1)", double(p));
  FSB_REQUIRE(p == 0.f || stream_base != nullptr, "dropout: p > 0 needs the device stream counter");
  FSB_REQUIRE(site >= 0, "dropout: negative site");
  d->seed = seed;
  d->stream_base = stream_base;
  d->site = site;
  d->thr = uint32_t(p * 256.f + 0.5f);
  d->keep_scale = 1.f / (1.f - p);
  return FSB_OK;
}

struct DropKey {
  uint32_t k0, k1, s_lo, s_hi, thr;
};
__device__ __forceinline__ DropKey drop_key(const DropArgs& d) {
  const uint64_t s = uint64_t(*d.stream_base + d.site);
  return DropKey{uint32_t(d.seed), uint32_t(d.seed >> 32), uint32_t(s), uint32_t(s >> 32), d.thr};
}
__device__ __forceinline__ bool drop_keep(uint32_t word, int byte, uint32_t thr) { return ((word >> (8 * byte)) & 0xffu) >= thr; }

// Hidden dropout, element (row, col): counter (col / 16, row, stream lo, stream hi); byte col % 16 of the output (word
// (col % 16) / 4, bits 8 (col % 4)).
__device__ __forceinline__ uint4 drop_hidden_bits(const DropKey& k, uint32_t row, uint32_t col16) {
  return philox4x32_10(make_uint4(col16, row, k.s_lo, k.s_hi), k.k0, k.k1);
}

// The hidden-layout keep bits of the 8 columns 8 c .. 8 c + 7 of `row` (bit j: column 8 c + j). One Philox call covers 16
// columns; this vector uses half of it. Everything arrives by value: the seed, threshold and scale straight from the kernel
// parameters (constant bank), the stream from the one load each thread makes before its loop — no copy of the parameter
// struct is ever addressed.
__device__ __forceinline__ uint32_t keep_bits8(uint64_t seed, uint32_t s_lo, uint32_t s_hi, uint32_t thr, int row, int c) {
  const DropKey k{uint32_t(seed), uint32_t(seed >> 32), s_lo, s_hi, thr};
  const uint4 r = drop_hidden_bits(k, uint32_t(row), uint32_t(c >> 1));
  const uint32_t w0 = (c & 1) ? r.z : r.x, w1 = (c & 1) ? r.w : r.y;
  uint32_t bits = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) bits |= uint32_t(drop_keep(j < 4 ? w0 : w1, j & 3, thr)) << j;
  return bits;
}
// x *= Z / (1 - p) over the 8 columns of keep_bits8
__device__ __forceinline__ void apply_keep8(uint32_t bits, float keep_scale, float (&x)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] = (bits >> j) & 1u ? x[j] * keep_scale : 0.f;
}
// the stream number s = *stream_base + site of a dropout site, split in halves (0 without dropout: nothing is read)
template <bool kDrop>
__device__ __forceinline__ void drop_stream(const int64_t* stream_base, int64_t site, uint32_t& s_lo, uint32_t& s_hi) {
  s_lo = s_hi = 0;
  if constexpr (kDrop) {
    const uint64_t s = uint64_t(*stream_base + site);
    s_lo = uint32_t(s);
    s_hi = uint32_t(s >> 32);
  }
}

// Attention dropout, element (b, head, q, k), with q = 16 qa + 8 qh + 2 qs + qp and k = 16 ka + 8 kh + 2 ks + kp:
// counter ((ka * 4 + ks) | (qa * 4 + qs) << 16, b * nheads + head, stream lo, stream hi); word 2 qp + kp, byte 2 qh + kh.
// One call covers the 4 x 4 block q in {16 qa + 2 qs + {0, 1, 8, 9}}, k likewise. In the wgmma accumulator layout a thread owns
// the two rows {r, r + 8} and column pairs {c, c + 1} of every 8-column group, so a thread of the row-major kernels (forward, dQ)
// needs the two words of its qp and a thread of the transposed dKV kernel the two words of its kp; lanes L and L ^ 4 need the
// other two words of the same call. Each pair of lanes therefore computes one call per block pair and swaps half of it
// (attn_drop_rows / attn_drop_cols): both orientations use every Philox output, none is computed twice.
__device__ __forceinline__ uint4 drop_attn_call(const DropKey& k, uint32_t bh, uint32_t qc, uint32_t kc) {
  return philox4x32_10(make_uint4(kc | (qc << 16), bh, k.s_lo, k.s_hi), k.k0, k.k1);
}

// Row-major fragment (rows q_r and q_r + 8 with q_r % 16 == lane / 4; columns c0 + 8 i + 2 (lane % 4) + e, c0 % 16 == 0).
// w[m][kp] = the word of column group pair m (columns c0 + 16 m + ...) holding this thread's bits: byte 2 qh + kh, where
// qh is the row half and kh = i % 2 for i = 2 m + kh.
template <int NM>
__device__ __forceinline__ void attn_drop_rows(const DropKey& k, uint32_t bh, int q_r, int c0, int lane, uint32_t (&w)[NM][2]) {
  const uint32_t qp = (lane >> 2) & 1, ks = lane & 3;
  const uint32_t qc = uint32_t(q_r >> 4) * 4 + ((q_r >> 1) & 3);
#pragma unroll
  for (int m = 0; m < NM; m += 2) {
    const uint32_t ka = uint32_t((c0 >> 4) + m + qp);          // this lane computes block m + qp, its partner m + 1 - qp
    const uint4 r = drop_attn_call(k, bh, qc, ka * 4 + ks);
    const uint32_t give0 = qp ? r.x : r.z, give1 = qp ? r.y : r.w;   // the partner's words (its qp = 1 - qp)
    const uint32_t own0 = qp ? r.z : r.x, own1 = qp ? r.w : r.y;
    const uint32_t got0 = __shfl_xor_sync(0xffffffffu, give0, 4), got1 = __shfl_xor_sync(0xffffffffu, give1, 4);
    w[m][0] = qp ? got0 : own0; w[m][1] = qp ? got1 : own1;   // selects, not a register index that depends on the lane
    w[m + 1][0] = qp ? own0 : got0; w[m + 1][1] = qp ? own1 : got1;
  }
}

// Transposed fragment of the dKV kernel (key rows k_r and k_r + 8 with k_r % 16 == lane / 4; query columns
// c0 + 8 i + 2 (lane % 4) + c, c0 % 16 == 0). w[m][qp] = the word of query group pair m for this thread's kp; byte 2 qh + kh
// with qh = i % 2 and kh the key-row half.
template <int NM>
__device__ __forceinline__ void attn_drop_cols(const DropKey& k, uint32_t bh, int k_r, int c0, int lane, uint32_t (&w)[NM][2]) {
  const uint32_t kp = (lane >> 2) & 1, qs = lane & 3;
  const uint32_t kc = uint32_t(k_r >> 4) * 4 + ((k_r >> 1) & 3);
#pragma unroll
  for (int m = 0; m < NM; m += 2) {
    const uint32_t qa = uint32_t((c0 >> 4) + m + kp);
    const uint4 r = drop_attn_call(k, bh, qa * 4 + qs, kc);
    // words 2 qp + kp: this lane keeps (kp, 2 + kp), the partner needs (1 - kp, 3 - kp)
    const uint32_t give0 = kp ? r.x : r.y, give1 = kp ? r.z : r.w;
    const uint32_t own0 = kp ? r.y : r.x, own1 = kp ? r.w : r.z;
    const uint32_t got0 = __shfl_xor_sync(0xffffffffu, give0, 4), got1 = __shfl_xor_sync(0xffffffffu, give1, 4);
    w[m][0] = kp ? got0 : own0; w[m][1] = kp ? got1 : own1;   // selects, not a register index that depends on the lane
    w[m + 1][0] = kp ? own0 : got0; w[m + 1][1] = kp ? own1 : got1;
  }
}

// attn_drop_cols compressed to one register: bit 4 i + 2 kh + qp is the keep bit of query pair i (qh = i % 2, group pair
// i / 2), key-row half kh and query parity qp — the accumulator index 4 i + e of the transposed fragment (e = 2 kh + qp).
template <int NM>
__device__ __forceinline__ uint32_t attn_keep_cols(const DropKey& k, uint32_t bh, int k_r, int c0, int lane) {
  static_assert(NM * 2 * 4 <= 32, "one bit per element of a thread's fragment");
  uint32_t bits = 0;
#pragma unroll
  for (int m = 0; m < NM; m += 2) {
    uint32_t w[2][2];
    attn_drop_cols<2>(k, bh, k_r, c0 + 16 * m, lane, w);
#pragma unroll
    for (int mm = 0; mm < 2; ++mm)
#pragma unroll
      for (int qh = 0; qh < 2; ++qh)
#pragma unroll
        for (int kh = 0; kh < 2; ++kh)
#pragma unroll
          for (int qp = 0; qp < 2; ++qp)
            bits |= uint32_t(drop_keep(w[mm][qp], 2 * qh + kh, k.thr)) << (4 * (2 * (m + mm) + qh) + 2 * kh + qp);
  }
  return bits;
}

}  // namespace fsb
