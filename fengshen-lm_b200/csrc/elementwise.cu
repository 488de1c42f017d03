// fsb200 — HBM-bound pointwise / gather kernels of the step. All bf16 I/O with fp32 math, 16-byte vector accesses,
// grid-stride loops with grid = k * #SMs.
//   rope        : layers/positional_embeddings.py:71-87 (rotate_half convention) applied in place to the q and k
//                 slices of the packed QKV projection output (layers/transformer.py:488-523)
//   swiglu      : LLaMAParallelMLP.forward layers/transformer.py:620-623  silu(w1 x) * (w3 x)
//   gated gelu  : MT5DenseGatedActDense (transformers mt5/modeling_mt5.py:96-123)  gelu_new(wi_0 x) * (wi_1 x)
//   gelu fwd/bwd: layers/activations.py:60-94 (tanh form, hand-written backward) and :98-117 (erf form)
//   embedding   : VocabParallelEmbedding.forward mpu/layers.py:104-130 (+ learned position / token-type rows for
//                 BERT / GPT-2: transformers bert/modeling_bert.py:53-112, gpt2/modeling_gpt2.py wte+wpe)
//   add         : residual adds layers/transformer.py:775-788
//   dropout     : y = x * Z / (1 - p) with the hidden-dropout mask of philox.cuh (BERT / MegatronBERT / mT5 embedding sites)
#include "host_common.h"
#include "philox.cuh"
#include "ptx.cuh"

namespace fsb {

static int ew_grid(int64_t work_items, int threads) {
  int64_t blocks = (work_items + threads - 1) / threads;
  int64_t cap = int64_t(num_sms()) * 16;
  return int(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

// ---------------------------------------------------------------------------------------------- rope
// x: rows of `nheads` heads; head h of row t starts at x + t*row_stride + h*head_stride (elements); head_dim D.
// Rotates D/2 pairs (d, d+D/2): out_d = x_d cos - sign*x_{d+D/2} sin ; out_{d+D/2} = x_{d+D/2} cos + sign*x_d sin.
// cos/sin: fp32 tables [max_pos, D/2]; pos[t] int64 (position_ids flattened to rows).  sign=+1 fwd, -1 bwd.
__global__ void __launch_bounds__(256) rope_kernel(__nv_bfloat16* __restrict__ x, const float* __restrict__ cos_t,
                                                   const float* __restrict__ sin_t, const int64_t* __restrict__ pos,
                                                   int64_t rows, int nheads, int D, int64_t row_stride,
                                                   int64_t head_stride, float sign, int64_t max_pos) {
  const int half = D >> 1;
  const int vec_per_head = half >> 3;  // 8 pairs per thread-iteration
  const int64_t total = rows * nheads * vec_per_head;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int v = int(i % vec_per_head);
    const int64_t th = i / vec_per_head;
    const int h = int(th % nheads);
    const int64_t t = th / nheads;
    const int64_t p = pos[t];
    __nv_bfloat16* base = x + t * row_stride + h * head_stride + v * 8;
    if (p < 0 || p >= max_pos) {
      // a position outside the cos/sin table (the reference regrows its cache, positional_embeddings.py:54-68; the host
      // wrapper sizes the table and validates position_ids): never read out of bounds — poison the row so the loss is NaN
      const uint32_t nan2 = 0x7fc07fc0u;
      *reinterpret_cast<uint4*>(base) = make_uint4(nan2, nan2, nan2, nan2);
      *reinterpret_cast<uint4*>(base + half) = make_uint4(nan2, nan2, nan2, nan2);
      continue;
    }
    float a[8], b[8], c[8], s[8];
    unpack8(*reinterpret_cast<const uint4*>(base), a);
    unpack8(*reinterpret_cast<const uint4*>(base + half), b);
    const float4* cp = reinterpret_cast<const float4*>(cos_t + p * half + v * 8);
    const float4* sp = reinterpret_cast<const float4*>(sin_t + p * half + v * 8);
    float4 c0 = cp[0], c1 = cp[1], s0 = sp[0], s1 = sp[1];
    c[0] = c0.x; c[1] = c0.y; c[2] = c0.z; c[3] = c0.w; c[4] = c1.x; c[5] = c1.y; c[6] = c1.z; c[7] = c1.w;
    s[0] = s0.x; s[1] = s0.y; s[2] = s0.z; s[3] = s0.w; s[4] = s1.x; s[5] = s1.y; s[6] = s1.z; s[7] = s1.w;
    float oa[8], ob[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      oa[j] = a[j] * c[j] - sign * b[j] * s[j];
      ob[j] = b[j] * c[j] + sign * a[j] * s[j];
    }
    *reinterpret_cast<uint4*>(base) = pack8(oa);
    *reinterpret_cast<uint4*>(base + half) = pack8(ob);
  }
}

// ---------------------------------------------------------------------------------------------- gated activations
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  return 0.5f * x * (1.f + tanhf(k0 * x * (1.f + k1 * x * x)));
}
__device__ __forceinline__ float dgelu_tanh_f(float x) {
  // activations.py:70-77 bias_gelu_back
  const float t = tanhf(0.79788456f * x * (1.f + 0.044715f * x * x));
  return 0.5f * x * ((1.f - t * t) * (0.79788456f + 0.1070322243f * x * x)) + 0.5f * (1.f + t);
}
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.f + erff(x * 0.7071067811865476f)); }
__device__ __forceinline__ float dgelu_erf_f(float x) {
  return 0.5f * (1.f + erff(x * 0.7071067811865476f)) + x * 0.3989422804014327f * __expf(-0.5f * x * x);
}
// act: 0 silu, 1 gelu_tanh, 2 gelu_erf, 3 tanh (BERT pooler, transformers bert/modeling_bert.py BertPooler)
template <int ACT>
__device__ __forceinline__ float act_f(float x) {
  if (ACT == 0) return x * sigmoid_f(x);
  if (ACT == 1) return gelu_tanh_f(x);
  if (ACT == 2) return gelu_erf_f(x);
  return tanhf(x);
}
template <int ACT>
__device__ __forceinline__ float dact_f(float x) {
  if (ACT == 0) { float s = sigmoid_f(x); return s * (1.f + x * (1.f - s)); }
  if (ACT == 1) return dgelu_tanh_f(x);
  if (ACT == 2) return dgelu_erf_f(x);
  const float t = tanhf(x);
  return 1.f - t * t;
}

// out[t, c] = act(gate[t, c]) * up[t, c]; gate/up/out have independent row strides (elements).
// kDrop: out[t, c] = act(gate[t, c]) * up[t, c] * Z / (1 - p), Z the hidden-dropout mask of philox.cuh at (t, c) of out; the
// backward applies the same mask to dout first (MT5DenseGatedActDense's dropout between the product and wo).
template <int ACT, bool kDrop>
__global__ void __launch_bounds__(256) glu_fwd_kernel(const __nv_bfloat16* __restrict__ gate,
                                                      const __nv_bfloat16* __restrict__ up,
                                                      __nv_bfloat16* __restrict__ out, int64_t rows, int cols,
                                                      int64_t ld_gate, int64_t ld_up, int64_t ld_out, const DropArgs drop) {
  const int vpr = cols >> 3;
  const int64_t total = rows * vpr;
  uint32_t s_lo, s_hi;
  drop_stream<kDrop>(drop.stream_base, drop.site, s_lo, s_hi);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t t = i / vpr;
    const int c = int(i % vpr) * 8;
    float g[8], u[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(gate + t * ld_gate + c), g);
    unpack8(*reinterpret_cast<const uint4*>(up + t * ld_up + c), u);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = act_f<ACT>(g[j]) * u[j];
    if constexpr (kDrop) apply_keep8(keep_bits8(drop.seed, s_lo, s_hi, drop.thr, int(t), c >> 3), drop.keep_scale, o);
    *reinterpret_cast<uint4*>(out + t * ld_out + c) = pack8(o);
  }
}
template <int ACT, bool kDrop>
__global__ void __launch_bounds__(256) glu_bwd_kernel(const __nv_bfloat16* __restrict__ dout,
                                                      const __nv_bfloat16* __restrict__ gate,
                                                      const __nv_bfloat16* __restrict__ up,
                                                      __nv_bfloat16* __restrict__ dgate, __nv_bfloat16* __restrict__ dup,
                                                      int64_t rows, int cols, int64_t ld_dout, int64_t ld_gate,
                                                      int64_t ld_up, int64_t ld_dgate, int64_t ld_dup, const DropArgs drop) {
  const int vpr = cols >> 3;
  const int64_t total = rows * vpr;
  uint32_t s_lo, s_hi;
  drop_stream<kDrop>(drop.stream_base, drop.site, s_lo, s_hi);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t t = i / vpr;
    const int c = int(i % vpr) * 8;
    float d[8], g[8], u[8], og[8], ou[8];
    unpack8(*reinterpret_cast<const uint4*>(dout + t * ld_dout + c), d);
    if constexpr (kDrop) apply_keep8(keep_bits8(drop.seed, s_lo, s_hi, drop.thr, int(t), c >> 3), drop.keep_scale, d);
    unpack8(*reinterpret_cast<const uint4*>(gate + t * ld_gate + c), g);
    unpack8(*reinterpret_cast<const uint4*>(up + t * ld_up + c), u);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      og[j] = d[j] * u[j] * dact_f<ACT>(g[j]);
      ou[j] = d[j] * act_f<ACT>(g[j]);
    }
    *reinterpret_cast<uint4*>(dgate + t * ld_dgate + c) = pack8(og);
    *reinterpret_cast<uint4*>(dup + t * ld_dup + c) = pack8(ou);
  }
}

// Plain activation: y = act(x) ; backward dx = dy * act'(x). Contiguous [n] (n % 8 == 0).
template <int ACT>
__global__ void __launch_bounds__(256) act_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int64_t nvec) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < nvec; i += int64_t(gridDim.x) * blockDim.x) {
    float a[8], o[8];
    unpack8(x[i], a);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = act_f<ACT>(a[j]);
    y[i] = pack8(o);
  }
}
template <int ACT>
__global__ void __launch_bounds__(256) act_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x,
                                                      uint4* __restrict__ dx, int64_t nvec) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < nvec; i += int64_t(gridDim.x) * blockDim.x) {
    float a[8], d[8], o[8];
    unpack8(x[i], a);
    unpack8(dy[i], d);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = d[j] * dact_f<ACT>(a[j]);
    dx[i] = pack8(o);
  }
}

// out = a + b (bf16, contiguous)
__global__ void __launch_bounds__(256) add_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b,
                                                  uint4* __restrict__ out, int64_t nvec) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < nvec; i += int64_t(gridDim.x) * blockDim.x) {
    float x[8], y[8], o[8];
    unpack8(a[i], x);
    unpack8(b[i], y);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = x[j] + y[j];
    out[i] = pack8(o);
  }
}

// x *= *scale (device scalar); exits without touching memory when *scale == 1 (the usual upstream gradient of a loss)
__global__ void __launch_bounds__(256) scale_inplace_kernel(uint4* __restrict__ x, int64_t nvec,
                                                            const float* __restrict__ scale) {
  const float s = *scale;
  if (s == 1.0f) return;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < nvec; i += int64_t(gridDim.x) * blockDim.x) {
    float f[8];
    unpack8(x[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= s;
    x[i] = pack8(f);
  }
}

// y = x * Z / (1 - p) over [rows, cols]; one thread per 16-column group = one Philox call. The same op is the backward
// (dx = dy * Z / (1 - p)).
__global__ void __launch_bounds__(256) dropout_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int64_t rows,
                                                      int cols, const DropArgs drop) {
  const int nvec = cols >> 3, ngrp = (nvec + 1) >> 1;
  const DropKey k = drop_key(drop);
  for (int64_t g = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; g < rows * ngrp; g += int64_t(gridDim.x) * blockDim.x) {
    const int64_t row = g / ngrp;
    const int c16 = int(g - row * ngrp);
    const uint4 r = drop_hidden_bits(k, uint32_t(row), uint32_t(c16));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = 2 * c16 + h;
      if (c >= nvec) break;
      const uint32_t w0 = h ? r.z : r.x, w1 = h ? r.w : r.y;
      float f[8];
      unpack8(x[row * nvec + c], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = drop_keep(j < 4 ? w0 : w1, j & 3, k.thr) ? f[j] * drop.keep_scale : 0.f;
      y[row * nvec + c] = pack8(f);
    }
  }
}

// saved = *base; *base += n — the dropout stream counter, advanced on the device once per training forward
__global__ void dropout_advance_kernel(int64_t* __restrict__ base, int64_t* __restrict__ saved, int64_t n) {
  const int64_t b = *base;
  *saved = b;
  *base = b + n;
}

// acc (fp32) += scale * x (bf16)   — gradient accumulation into the fp32 shard (ZeRO-2 per-micro-step reduce)
__global__ void __launch_bounds__(256) accumulate_kernel(float* __restrict__ acc, const uint2* __restrict__ x,
                                                         int64_t nvec, float scale, int overwrite) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < nvec; i += int64_t(gridDim.x) * blockDim.x) {
    const uint2 q = x[i];
    float4 a = overwrite ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<float4*>(acc)[i];
    a.x += scale * bf16lo(q.x); a.y += scale * bf16hi(q.x); a.z += scale * bf16lo(q.y); a.w += scale * bf16hi(q.y);
    reinterpret_cast<float4*>(acc)[i] = a;
  }
}

// Column sums of a bf16 matrix x[rows, cols] (row stride ld): bias gradients db[n] = sum_t dy[t, n], and the learned
// position-embedding gradient dP[s,:] = sum_b dx[b,s,:] (view x as [B, S*h]). Stage 1: each CTA sums a strip of rows for
// a 256-column tile (8 columns per thread, 32 row-lanes) -> partial[strip, cols] fp32; stage 2 reduces the strips.
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ partial,
                                                          int64_t rows, int cols, int64_t ld, int rows_per_strip) {
  __shared__ float sm[8][64 + 1];  // [row-lane][col within tile]; 8 lanes x 64 cols per CTA
  const int cl = threadIdx.x & 7;        // 8 threads x 8 cols = 64 columns per CTA
  const int rl = threadIdx.x >> 3;       // 32 row lanes
  const int col = blockIdx.x * 64 + cl * 8;
  const int64_t r0 = int64_t(blockIdx.y) * rows_per_strip;
  const int64_t r1 = min(rows, r0 + rows_per_strip);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (col < cols) {
    for (int64_t r = r0 + rl; r < r1; r += 32) {
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>(x + r * ld + col), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
  }
  // reduce the 32 row lanes: first within each warp (4 row lanes per warp: lanes differ in bits 3,4), then via smem
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 8);
    acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 16);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) < 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) sm[w][cl * 8 + j] = acc[j];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x];
    const int c = blockIdx.x * 64 + threadIdx.x;
    if (c < cols) partial[int64_t(blockIdx.y) * cols + c] = t;
  }
}
// dx = dy * act'(x) AND partial column sums of dx in the same pass (the bias gradient of the linear layer that produced x).
// A CTA owns 256 columns x a strip of rows: every warp streams whole 512-byte row segments (three streams: x, dy, dx), two rows
// in flight per thread; the 8 row lanes are combined through shared memory and written as partial[strip, cols].
template <int ACT>
__global__ void __launch_bounds__(256) act_bwd_colsum_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                             __nv_bfloat16* __restrict__ dx, float* __restrict__ partial,
                                                             int64_t rows, int cols, int rows_per_strip) {
  __shared__ float sm[8][256 + 4];
  const int cl = threadIdx.x & 31;
  const int rl = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + cl * 8;
  const int64_t r0 = int64_t(blockIdx.y) * rows_per_strip;
  const int64_t r1 = min(rows, r0 + rows_per_strip);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (col < cols) {
    for (int64_t r = r0 + rl; r < r1; r += 16) {
      const bool two = r + 8 < r1;
      const uint4 xa = *reinterpret_cast<const uint4*>(x + r * cols + col);
      const uint4 da = *reinterpret_cast<const uint4*>(dy + r * cols + col);
      uint4 xb = make_uint4(0, 0, 0, 0), db = make_uint4(0, 0, 0, 0);
      if (two) {
        xb = *reinterpret_cast<const uint4*>(x + (r + 8) * cols + col);
        db = *reinterpret_cast<const uint4*>(dy + (r + 8) * cols + col);
      }
      float a[8], d[8], o[8], f[8];
      unpack8(xa, a); unpack8(da, d);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = d[j] * dact_f<ACT>(a[j]);
      uint4 q = pack8(o);
      *reinterpret_cast<uint4*>(dx + r * cols + col) = q;
      unpack8(q, f);   // sum what was stored (bf16-rounded): exactly what a separate colsum over dx would add up
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
      if (two) {
        unpack8(xb, a); unpack8(db, d);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = d[j] * dact_f<ACT>(a[j]);
        q = pack8(o);
        *reinterpret_cast<uint4*>(dx + (r + 8) * cols + col) = q;
        unpack8(q, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sm[rl][cl * 8 + j] = acc[j];
  __syncthreads();
  {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x];
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c < cols) partial[int64_t(blockIdx.y) * cols + c] = t;
  }
}
__global__ void __launch_bounds__(256) colsum_finish_kernel(const float* __restrict__ partial, void* __restrict__ out,
                                                            int nparts, int cols, int out_f32, int accumulate) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= cols) return;
  float t = 0.f;
  for (int r = 0; r < nparts; ++r) t += partial[int64_t(r) * cols + c];
  if (out_f32) {
    float* o = reinterpret_cast<float*>(out);
    o[c] = accumulate ? o[c] + t : t;
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
    o[c] = __float2bfloat16(accumulate ? __bfloat162float(o[c]) + t : t);
  }
}

// ---------------------------------------------------------------------------------------------- embedding
// out[t] = W[ids[t]] (+ P[pos[t]]) (+ T[tt[t]]);   pos == nullptr with P != nullptr means pos[t] = t % seq_len.
__global__ void __launch_bounds__(256) embedding_fwd_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ pos,
                                                            const int64_t* __restrict__ tt,
                                                            const __nv_bfloat16* __restrict__ W,
                                                            const __nv_bfloat16* __restrict__ P,
                                                            const __nv_bfloat16* __restrict__ T,
                                                            __nv_bfloat16* __restrict__ out, int64_t rows, int cols,
                                                            int seq_len) {
  const int vpr = cols >> 3;
  const int64_t total = rows * vpr;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t t = i / vpr;
    const int c = int(i % vpr) * 8;
    float o[8];
    unpack8(*reinterpret_cast<const uint4*>(W + ids[t] * cols + c), o);
    if (P != nullptr) {
      const int64_t p = pos ? pos[t] : (t % seq_len);
      float a[8];
      unpack8(*reinterpret_cast<const uint4*>(P + p * cols + c), a);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] += a[j];
    }
    if (T != nullptr) {
      float a[8];
      unpack8(*reinterpret_cast<const uint4*>(T + (tt ? tt[t] : 0) * cols + c), a);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] += a[j];
    }
    *reinterpret_cast<uint4*>(out + t * cols + c) = pack8(o);
  }
}
// dW[ids[t]] += dout[t]  (bf16x2 reductions at L2; rows hit by several tokens accumulate there)
__global__ void __launch_bounds__(256) embedding_bwd_kernel(const int64_t* __restrict__ ids,
                                                            const __nv_bfloat16* __restrict__ dout,
                                                            __nv_bfloat16* __restrict__ dW, int64_t rows, int cols,
                                                            int64_t idx_mod) {
  const int vpr = cols >> 3;
  const int64_t total = rows * vpr;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t t = i / vpr;
    const int c = int(i % vpr) * 8;
    const int64_t r = ids ? ids[t] : (t % idx_mod);
    const uint4 q = *reinterpret_cast<const uint4*>(dout + t * cols + c);
    __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>(dW + r * cols + c);
    atomicAdd(dst + 0, *reinterpret_cast<const __nv_bfloat162*>(&q.x));
    atomicAdd(dst + 1, *reinterpret_cast<const __nv_bfloat162*>(&q.y));
    atomicAdd(dst + 2, *reinterpret_cast<const __nv_bfloat162*>(&q.z));
    atomicAdd(dst + 3, *reinterpret_cast<const __nv_bfloat162*>(&q.w));
  }
}


// Deterministic embedding backward. `ids_sorted` / `order` are the token ids sorted ascending (stable) and the token index
// of each sorted position. One CTA per sorted position; only the CTA at the START of a run of equal ids works: it sums the
// run's dout rows in fp32 — EMB_R occurrences in flight (occurrence j goes to sub-sum j % EMB_R), combined in a fixed order —
// and adds the total onto dW[id] with ONE bf16 rounding. torch's embedding backward (what the reference runs) accumulates
// in fp32 as well; the former bf16x2 atomics rounded after every occurrence and depended on the atomic order.
constexpr int EMB_R = 4;
__global__ void __launch_bounds__(256) embedding_bwd_sorted_kernel(const int64_t* __restrict__ ids_sorted,
                                                                   const int64_t* __restrict__ order,
                                                                   const __nv_bfloat16* __restrict__ dout,
                                                                   __nv_bfloat16* __restrict__ dW, int64_t rows, int cols) {
  const int64_t i0 = blockIdx.x;
  const int64_t id = ids_sorted[i0];
  if (i0 > 0 && ids_sorted[i0 - 1] == id) return;   // not the start of a run
  __shared__ float red[EMB_R][64 * 8];
  const int lane_c = threadIdx.x & 63, r = threadIdx.x >> 6;   // 64 column vectors x EMB_R occurrences in flight
  const int vpr = cols >> 3;
  for (int cv0 = 0; cv0 < vpr; cv0 += 64) {
    const int cv = cv0 + lane_c;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (cv < vpr) {
      for (int64_t j = i0 + r; j < rows && ids_sorted[j] == id; j += EMB_R) {
        float f[8];
        unpack8(*reinterpret_cast<const uint4*>(dout + order[j] * cols + cv * 8), f);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += f[e];
      }
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 8; ++e) red[r][lane_c * 8 + e] = acc[e];
    __syncthreads();
    if (r == 0 && cv < vpr) {
      float f[8];
      __nv_bfloat16* dst = dW + id * cols + cv * 8;
      unpack8(*reinterpret_cast<const uint4*>(dst), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float t = red[0][lane_c * 8 + e];
#pragma unroll
        for (int q = 1; q < EMB_R; ++q) t += red[q][lane_c * 8 + e];
        f[e] += t;
      }
      *reinterpret_cast<uint4*>(dst) = pack8(f);
    }
  }
}

// out (bf16) = in (fp32), 8 elements per thread-iteration
__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out,
                                                            int64_t n8) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n8; i += int64_t(gridDim.x) * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(in)[2 * i], b = reinterpret_cast<const float4*>(in)[2 * i + 1];
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    reinterpret_cast<uint4*>(out)[i] = pack8(f);
  }
}

}  // namespace fsb

using namespace fsb;

extern "C" int fsb_embedding_bwd_sorted(const int64_t* ids_sorted, const int64_t* order, const void* dout, void* dW,
                                        int64_t rows, int64_t cols, fsb_stream_t st) {
  FSB_REQUIRE(ids_sorted && order && dout && dW && rows > 0 && cols > 0 && cols % 8 == 0, "embedding_bwd_sorted: bad args");
  FSB_REQUIRE(rows < (int64_t(1) << 31), "embedding_bwd_sorted: too many rows");
  FSB_REQUIRE(aligned16(dout) && aligned16(dW), "embedding_bwd_sorted: alignment");
  embedding_bwd_sorted_kernel<<<unsigned(rows), 256, 0, (cudaStream_t)st>>>(
      ids_sorted, order, (const __nv_bfloat16*)dout, (__nv_bfloat16*)dW, rows, int(cols));
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

extern "C" int fsb_cast_f32_to_bf16(const float* in, void* out, int64_t n, fsb_stream_t st) {
  FSB_REQUIRE(in && out && n > 0 && n % 8 == 0, "cast_f32_to_bf16: n must be a positive multiple of 8");
  FSB_REQUIRE(aligned16(in) && aligned16(out), "cast_f32_to_bf16: alignment");
  cast_f32_bf16_kernel<<<ew_grid(n / 8, 256), 256, 0, (cudaStream_t)st>>>(in, (__nv_bfloat16*)out, n / 8);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

extern "C" int fsb_rope_inplace(void* x, const float* cos_table, const float* sin_table, const int64_t* positions,
                                int64_t rows, int nheads, int head_dim, int64_t row_stride, int64_t head_stride,
                                int64_t max_pos, int backward, fsb_stream_t st) {
  FSB_REQUIRE(x && cos_table && sin_table && positions, "rope: null pointer");
  FSB_REQUIRE(rows > 0 && nheads > 0 && head_dim % 16 == 0 && head_dim > 0, "rope: head_dim must be a multiple of 16");
  FSB_REQUIRE(row_stride % 8 == 0 && head_stride % 8 == 0 && aligned16(x) && aligned16(cos_table) && aligned16(sin_table),
              "rope: alignment");
  FSB_REQUIRE(max_pos > 0, "rope: max_pos (rows of the cos/sin tables) must be positive");
  const int64_t total = rows * nheads * (head_dim / 16);
  rope_kernel<<<ew_grid(total, 256), 256, 0, (cudaStream_t)st>>>((__nv_bfloat16*)x, cos_table, sin_table, positions, rows,
                                                               nheads, head_dim, row_stride, head_stride,
                                                               backward ? -1.f : 1.f, max_pos);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

static int glu_fwd(int act, const void* gate, const void* up, void* out, int64_t rows, int64_t cols, int64_t ld_gate,
                   int64_t ld_up, int64_t ld_out, const DropArgs* drop, cudaStream_t st) {
  FSB_REQUIRE(act >= 0 && act <= 2, "glu_fwd: bad act %d", act);
  FSB_REQUIRE(gate && up && out && rows > 0 && cols > 0 && cols % 8 == 0, "glu_fwd: bad args");
  FSB_REQUIRE(ld_gate % 8 == 0 && ld_up % 8 == 0 && ld_out % 8 == 0 && aligned16(gate) && aligned16(up) && aligned16(out),
              "glu_fwd: alignment");
  const int g = ew_grid(rows * (cols / 8), 256);
#define L(A, D) glu_fwd_kernel<A, D><<<g, 256, 0, st>>>((const __nv_bfloat16*)gate, (const __nv_bfloat16*)up,       \
                                                        (__nv_bfloat16*)out, rows, int(cols), ld_gate, ld_up, ld_out, \
                                                        drop ? *drop : DropArgs{})
  if (drop != nullptr) {
    if (act == 0) L(0, true); else if (act == 1) L(1, true); else L(2, true);
  } else {
    if (act == 0) L(0, false); else if (act == 1) L(1, false); else L(2, false);
  }
#undef L
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
static int glu_bwd(int act, const void* dout, const void* gate, const void* up, void* dgate, void* dup, int64_t rows,
                   int64_t cols, int64_t ld_dout, int64_t ld_gate, int64_t ld_up, int64_t ld_dgate, int64_t ld_dup,
                   const DropArgs* drop, cudaStream_t st) {
  FSB_REQUIRE(act >= 0 && act <= 2, "glu_bwd: bad act %d", act);
  FSB_REQUIRE(dout && gate && up && dgate && dup && rows > 0 && cols > 0 && cols % 8 == 0, "glu_bwd: bad args");
  FSB_REQUIRE((ld_dout | ld_gate | ld_up | ld_dgate | ld_dup) % 8 == 0 && aligned16(dout) && aligned16(gate) &&
                  aligned16(up) && aligned16(dgate) && aligned16(dup),
              "glu_bwd: alignment");
  const int g = ew_grid(rows * (cols / 8), 256);
#define L(A, D) glu_bwd_kernel<A, D><<<g, 256, 0, st>>>(                                                           \
      (const __nv_bfloat16*)dout, (const __nv_bfloat16*)gate, (const __nv_bfloat16*)up, (__nv_bfloat16*)dgate,       \
      (__nv_bfloat16*)dup, rows, int(cols), ld_dout, ld_gate, ld_up, ld_dgate, ld_dup, drop ? *drop : DropArgs{})
  if (drop != nullptr) {
    if (act == 0) L(0, true); else if (act == 1) L(1, true); else L(2, true);
  } else {
    if (act == 0) L(0, false); else if (act == 1) L(1, false); else L(2, false);
  }
#undef L
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_glu_fwd(int act, const void* gate, const void* up, void* out, int64_t rows, int64_t cols,
                           int64_t ld_gate, int64_t ld_up, int64_t ld_out, fsb_stream_t st) {
  return glu_fwd(act, gate, up, out, rows, cols, ld_gate, ld_up, ld_out, nullptr, (cudaStream_t)st);
}
extern "C" int fsb_glu_bwd(int act, const void* dout, const void* gate, const void* up, void* dgate, void* dup,
                           int64_t rows, int64_t cols, int64_t ld_dout, int64_t ld_gate, int64_t ld_up,
                           int64_t ld_dgate, int64_t ld_dup, fsb_stream_t st) {
  return glu_bwd(act, dout, gate, up, dgate, dup, rows, cols, ld_dout, ld_gate, ld_up, ld_dgate, ld_dup, nullptr,
                 (cudaStream_t)st);
}
extern "C" int fsb_glu_fwd_dropout(int act, const void* gate, const void* up, void* out, int64_t rows, int64_t cols,
                                   int64_t ld_gate, int64_t ld_up, int64_t ld_out, float p, uint64_t seed,
                                   const int64_t* stream_base, int64_t site, fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  if (p > 0.f) FSB_REQUIRE(rows <= 0x7fffffffll, "glu_fwd_dropout: more than 2^31 - 1 rows with p > 0");
  return glu_fwd(act, gate, up, out, rows, cols, ld_gate, ld_up, ld_out, p > 0.f ? &d : nullptr, (cudaStream_t)st);
}
extern "C" int fsb_glu_bwd_dropout(int act, const void* dout, const void* gate, const void* up, void* dgate, void* dup,
                                   int64_t rows, int64_t cols, int64_t ld_dout, int64_t ld_gate, int64_t ld_up,
                                   int64_t ld_dgate, int64_t ld_dup, float p, uint64_t seed, const int64_t* stream_base,
                                   int64_t site, fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  if (p > 0.f) FSB_REQUIRE(rows <= 0x7fffffffll, "glu_bwd_dropout: more than 2^31 - 1 rows with p > 0");
  return glu_bwd(act, dout, gate, up, dgate, dup, rows, cols, ld_dout, ld_gate, ld_up, ld_dgate, ld_dup,
                 p > 0.f ? &d : nullptr, (cudaStream_t)st);
}
extern "C" int fsb_act_fwd(int act, const void* x, void* y, int64_t n, fsb_stream_t st) {
  FSB_REQUIRE(act >= 0 && act <= 3 && x && y && n > 0 && n % 8 == 0 && aligned16(x) && aligned16(y), "act_fwd: bad args");
  const int g = ew_grid(n / 8, 256);
#define L(A) act_fwd_kernel<A><<<g, 256, 0, (cudaStream_t)st>>>((const uint4*)x, (uint4*)y, n / 8)
  if (act == 0) L(0); else if (act == 1) L(1); else if (act == 2) L(2); else L(3);
#undef L
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_act_bwd(int act, const void* dy, const void* x, void* dx, int64_t n, fsb_stream_t st) {
  FSB_REQUIRE(act >= 0 && act <= 3 && dy && x && dx && n > 0 && n % 8 == 0 && aligned16(x) && aligned16(dy) && aligned16(dx),
              "act_bwd: bad args");
  const int g = ew_grid(n / 8, 256);
#define L(A) act_bwd_kernel<A><<<g, 256, 0, (cudaStream_t)st>>>((const uint4*)dy, (const uint4*)x, (uint4*)dx, n / 8)
  if (act == 0) L(0); else if (act == 1) L(1); else if (act == 2) L(2); else L(3);
#undef L
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_add(const void* a, const void* b, void* out, int64_t n, fsb_stream_t st) {
  FSB_REQUIRE(a && b && out && n > 0 && n % 8 == 0 && aligned16(a) && aligned16(b) && aligned16(out), "add: bad args");
  add_kernel<<<ew_grid(n / 8, 256), 256, 0, (cudaStream_t)st>>>((const uint4*)a, (const uint4*)b, (uint4*)out, n / 8);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_scale_inplace(void* x, int64_t n, const float* scale_dev, fsb_stream_t st) {
  FSB_REQUIRE(x && scale_dev && n > 0 && n % 8 == 0 && aligned16(x), "scale_inplace: bad args (n %% 8 == 0, aligned)");
  scale_inplace_kernel<<<ew_grid(n / 8, 256), 256, 0, (cudaStream_t)st>>>((uint4*)x, n / 8, scale_dev);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_dropout(const void* x, void* y, int64_t rows, int64_t cols, float p, uint64_t seed,
                           const int64_t* stream_base, int64_t site, fsb_stream_t st) {
  FSB_REQUIRE(x && y && rows > 0 && cols > 0 && cols % 8 == 0 && cols <= (1 << 20) && aligned16(x) && aligned16(y),
              "dropout: bad args (cols %% 8 == 0, aligned)");
  FSB_REQUIRE(rows <= 0xffffffffll, "dropout: more than 2^32 rows");
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  if (p == 0.f) {
    if (x != y) {
      cudaError_t e = cudaMemcpyAsync(y, x, size_t(rows) * size_t(cols) * 2, cudaMemcpyDeviceToDevice, (cudaStream_t)st);
      if (e != cudaSuccess) {
        set_error("dropout: copy failed: %s", cudaGetErrorString(e));
        return FSB_ERR_CUDA;
      }
    }
    return FSB_OK;
  }
  const int64_t groups = rows * ((cols / 8 + 1) / 2);
  dropout_kernel<<<ew_grid(groups, 256), 256, 0, (cudaStream_t)st>>>((const uint4*)x, (uint4*)y, rows, int(cols), d);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_dropout_advance(int64_t* stream_base, int64_t* saved, int64_t n, fsb_stream_t st) {
  FSB_REQUIRE(stream_base && saved && n >= 0, "dropout_advance: bad args");
  dropout_advance_kernel<<<1, 1, 0, (cudaStream_t)st>>>(stream_base, saved, n);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
static void colsum_plan(int64_t rows, int64_t cols, int& nstrips, int& rows_per_strip) {
  const int col_tiles = int((cols + 63) / 64);
  int64_t want = (int64_t(4) * num_sms() + col_tiles - 1) / col_tiles;
  int64_t max_strips = (rows + 31) / 32;
  if (want > max_strips) want = max_strips;
  if (want < 1) want = 1;
  if (want > 1024) want = 1024;
  rows_per_strip = int(((rows + want - 1) / want + 31) / 32 * 32);
  nstrips = int((rows + rows_per_strip - 1) / rows_per_strip);
}
extern "C" size_t fsb_colsum_workspace_bytes(int64_t rows, int64_t cols) {
  int ns, rps;
  colsum_plan(rows, cols, ns, rps);
  return size_t(ns) * size_t(cols) * sizeof(float);
}
extern "C" int fsb_colsum(const void* x, int64_t rows, int64_t cols, int64_t ld, void* out, int out_dtype, int accumulate,
                          void* workspace, size_t workspace_bytes, fsb_stream_t st) {
  FSB_REQUIRE(x && out && workspace && rows > 0 && cols > 0 && cols % 8 == 0 && ld % 8 == 0 && aligned16(x),
              "colsum: bad args (cols, ld multiples of 8; 16-byte aligned)");
  int ns, rps;
  colsum_plan(rows, cols, ns, rps);
  FSB_REQUIRE(workspace_bytes >= size_t(ns) * cols * sizeof(float), "colsum: workspace too small");
  dim3 grid(unsigned((cols + 63) / 64), unsigned(ns));
  colsum_bf16_kernel<<<grid, 256, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)x, (float*)workspace, rows, int(cols), ld, rps);
  FSB_CUDA_LAUNCH_CHECK();
  colsum_finish_kernel<<<unsigned((cols + 255) / 256), 256, 0, (cudaStream_t)st>>>((const float*)workspace, out, ns,
                                                                                  int(cols), out_dtype == FSB_F32, accumulate);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
static void act_bwd_bias_plan(int64_t rows, int64_t cols, int& nstrips, int& rows_per_strip) {
  const int col_tiles = int((cols + 255) / 256);
  int64_t want = (int64_t(8) * num_sms() + col_tiles - 1) / col_tiles;
  const int64_t max_strips = (rows + 15) / 16;
  if (want > max_strips) want = max_strips;
  if (want < 1) want = 1;
  if (want > 2048) want = 2048;
  rows_per_strip = int(((rows + want - 1) / want + 15) / 16 * 16);
  nstrips = int((rows + rows_per_strip - 1) / rows_per_strip);
}
extern "C" size_t fsb_act_bwd_bias_workspace_bytes(int64_t rows, int64_t cols) {
  int ns, rps;
  act_bwd_bias_plan(rows, cols, ns, rps);
  return size_t(ns) * size_t(cols) * sizeof(float);
}
extern "C" int fsb_act_bwd_bias(int act, const void* dy, const void* x, void* dx, int64_t rows, int64_t cols, void* dbias,
                                int dbias_dtype, int accumulate, void* workspace, size_t workspace_bytes, fsb_stream_t st) {
  FSB_REQUIRE(dy && x && dx && dbias && workspace && rows > 0 && cols > 0 && cols % 8 == 0 && aligned16(dy) && aligned16(x) &&
                  aligned16(dx),
              "act_bwd_bias: bad args (cols multiple of 8; 16-byte aligned, contiguous rows)");
  FSB_REQUIRE(act >= 1 && act <= 3, "act_bwd_bias: act %d unsupported (1 tanh-GeLU, 2 erf-GeLU, 3 tanh)", act);
  int ns, rps;
  act_bwd_bias_plan(rows, cols, ns, rps);
  FSB_REQUIRE(workspace_bytes >= size_t(ns) * cols * sizeof(float), "act_bwd_bias: workspace too small");
  dim3 grid(unsigned((cols + 255) / 256), unsigned(ns));
  const __nv_bfloat16 *pdy = (const __nv_bfloat16*)dy, *px = (const __nv_bfloat16*)x;
  if (act == 1) act_bwd_colsum_kernel<1><<<grid, 256, 0, (cudaStream_t)st>>>(pdy, px, (__nv_bfloat16*)dx, (float*)workspace, rows, int(cols), rps);
  else if (act == 2) act_bwd_colsum_kernel<2><<<grid, 256, 0, (cudaStream_t)st>>>(pdy, px, (__nv_bfloat16*)dx, (float*)workspace, rows, int(cols), rps);
  else act_bwd_colsum_kernel<3><<<grid, 256, 0, (cudaStream_t)st>>>(pdy, px, (__nv_bfloat16*)dx, (float*)workspace, rows, int(cols), rps);
  FSB_CUDA_LAUNCH_CHECK();
  colsum_finish_kernel<<<unsigned((cols + 255) / 256), 256, 0, (cudaStream_t)st>>>((const float*)workspace, dbias, ns,
                                                                                  int(cols), dbias_dtype == FSB_F32, accumulate);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_accumulate(float* acc, const void* x, int64_t n, float scale, int overwrite, fsb_stream_t st) {
  FSB_REQUIRE(acc && x && n > 0 && n % 4 == 0 && aligned16(acc) && (reinterpret_cast<uintptr_t>(x) & 7) == 0,
              "accumulate: bad args (n %% 4 == 0, aligned)");
  accumulate_kernel<<<ew_grid(n / 4, 256), 256, 0, (cudaStream_t)st>>>(acc, (const uint2*)x, n / 4, scale, overwrite);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_embedding_fwd(const int64_t* ids, const int64_t* pos, const int64_t* token_type, const void* W,
                                 const void* P, const void* T, void* out, int64_t rows, int64_t cols, int64_t seq_len,
                                 fsb_stream_t st) {
  FSB_REQUIRE(ids && W && out && rows > 0 && cols > 0 && cols % 8 == 0 && seq_len > 0, "embedding_fwd: bad args");
  FSB_REQUIRE(aligned16(W) && aligned16(P) && aligned16(T) && aligned16(out), "embedding_fwd: alignment");
  embedding_fwd_kernel<<<ew_grid(rows * (cols / 8), 256), 256, 0, (cudaStream_t)st>>>(
      ids, pos, token_type, (const __nv_bfloat16*)W, (const __nv_bfloat16*)P, (const __nv_bfloat16*)T,
      (__nv_bfloat16*)out, rows, int(cols), int(seq_len));
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
extern "C" int fsb_embedding_bwd(const int64_t* ids, const void* dout, void* dW, int64_t rows, int64_t cols,
                                 int64_t idx_mod, fsb_stream_t st) {
  FSB_REQUIRE(dout && dW && rows > 0 && cols > 0 && cols % 8 == 0, "embedding_bwd: bad args");
  FSB_REQUIRE(ids != nullptr || idx_mod > 0, "embedding_bwd: need ids or idx_mod");
  FSB_REQUIRE(aligned16(dout) && aligned16(dW), "embedding_bwd: alignment");
  embedding_bwd_kernel<<<ew_grid(rows * (cols / 8), 256), 256, 0, (cudaStream_t)st>>>(
      ids, (const __nv_bfloat16*)dout, (__nv_bfloat16*)dW, rows, int(cols), idx_mod);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}
