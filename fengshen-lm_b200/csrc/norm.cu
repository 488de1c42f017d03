// fsb200 — RMSNorm / LayerNorm forward + backward (HBM-bound; one pass over each operand).
//   RMSNorm   : fengshen/models/megatron/layers/norms.py:44-52 (== MT5LayerNorm): y = scale * cast(x * rsqrt(mean(x^2)+eps))
//   LayerNorm : torch.nn.LayerNorm as re-exported at layers/norms.py:16 (BERT/GPT2/MegatronBERT via transformers)
// Optional fusions: residual add in forward (x_sum = x + residual is also written out), and "+= dres" in backward
// (gradient arriving through the residual branch), which removes the two un-fused adds at transformer.py:775-788.
// Layout: [rows, cols] bf16 row-major, cols % 8 == 0, cols <= 16384.
// Work split: a CTA of 256 threads holds RPC = 256/TPR rows at a time, TPR threads per row (TPR = 32..256 chosen so a
// thread owns <= 4 16-byte vectors; 768-wide rows use one warp per row, 5120-wide rows the whole CTA). The row lives in
// registers between the reduction and the normalisation, so x is read exactly once.
// Weight gradients: every thread accumulates fp32 partials over its rows; the CTA combines its RPC row slots through
// shared memory in a fixed order and writes partial[cta, cols]; a second kernel reduces the partials column-wise
// (deterministic, no atomics).
// Dropout on the branch (kDrop, with a residual only): the forward computes x_sum = x * Z / (1 - p) + residual, Z the
// hidden-dropout mask of philox.cuh at (row, col); the backward also writes dbranch = dx * Z / (1 - p) — the gradient of the
// dropped branch beside the gradient of the sum.
#include <stdlib.h>

#include "host_common.h"
#include "philox.cuh"
#include "ptx.cuh"

namespace fsb {

constexpr int NORM_THREADS = 256;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// dropout on norm rows is instantiated up to this many 8-column vectors per thread (cols <= 12288): wider rows already
// spill in the dropout-free backward
constexpr int NORM_DROP_MAX_VPT = 6;

// Sum of (a, b) over the TPR threads that share a row; result broadcast to those threads.
// red: [RPC][2][TPR/32] floats of shared memory. Every thread of the CTA must call (contains __syncthreads).
template <int TPR>
__device__ __forceinline__ void row_sum2(float& a, float& b, float* red, int row_slot, int lane_in_row) {
  a = warp_sum(a);
  b = warp_sum(b);
  if (TPR > 32) {
    constexpr int WPR = TPR / 32;
    const int w = lane_in_row >> 5;
    __syncthreads();
    if ((lane_in_row & 31) == 0) { red[(row_slot * 2 + 0) * WPR + w] = a; red[(row_slot * 2 + 1) * WPR + w] = b; }
    __syncthreads();
    float x = 0.f, y = 0.f;
#pragma unroll
    for (int i = 0; i < WPR; ++i) { x += red[(row_slot * 2 + 0) * WPR + i]; y += red[(row_slot * 2 + 1) * WPR + i]; }
    a = x; b = y;
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward.  kLayer = false: RMSNorm (stats[row] = rstd). kLayer = true: LayerNorm (stats[2*row] = mean, [2*row+1] = rstd)
// ------------------------------------------------------------------------------------------------------------
template <bool kLayer, int TPR, int VPT, bool kDrop>
__global__ void __launch_bounds__(NORM_THREADS) norm_fwd_kernel(
    const uint4* __restrict__ x, const uint4* __restrict__ residual, const uint4* __restrict__ gamma,
    const uint4* __restrict__ beta, uint4* __restrict__ y, uint4* __restrict__ sum_out, float* __restrict__ stats,
    int rows, int cols, float eps, const DropArgs drop) {
  constexpr int RPC = NORM_THREADS / TPR;
  __shared__ float red[RPC * 2 * (TPR / 32)];
  const int nvec = cols >> 3;
  const int row_slot = threadIdx.x / TPR, lir = threadIdx.x % TPR;
  uint32_t s_lo, s_hi;
  drop_stream<kDrop>(drop.stream_base, drop.site, s_lo, s_hi);
  for (int base_row = blockIdx.x * RPC; base_row < rows; base_row += gridDim.x * RPC) {
    const int row = base_row + row_slot;
    const bool rv = row < rows;
    const size_t base = size_t(row) * nvec;
    float xv[VPT][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = lir + i * TPR;
      if (rv && c < nvec) {
        unpack8(x[base + c], xv[i]);
        if (residual != nullptr) {
          float r[8];
          unpack8(residual[base + c], r);
          if constexpr (kDrop) apply_keep8(keep_bits8(drop.seed, s_lo, s_hi, drop.thr, row, c), drop.keep_scale, xv[i]);
#pragma unroll
          for (int j = 0; j < 8; ++j) xv[i][j] = round_bf16(xv[i][j] + r[j]);  // the sum lives in bf16 in the reference
          sum_out[base + c] = pack8(xv[i]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) { s1 += xv[i][j]; s2 += xv[i][j] * xv[i][j]; }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) xv[i][j] = 0.f;
      }
    }
    row_sum2<TPR>(s1, s2, red, row_slot, lir);
    float mean = 0.f, rstd;
    if (kLayer) {
      mean = s1 / cols;
      float v = 0.f, dummy = 0.f;  // two-pass variance from registers
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int c = lir + i * TPR;
        if (c < nvec) {
#pragma unroll
          for (int j = 0; j < 8; ++j) { const float d = xv[i][j] - mean; v += d * d; }
        }
      }
      row_sum2<TPR>(v, dummy, red, row_slot, lir);
      rstd = rsqrtf(v / cols + eps);
      if (rv && lir == 0) { stats[2 * row] = mean; stats[2 * row + 1] = rstd; }
    } else {
      rstd = rsqrtf(s2 / cols + eps);
      if (rv && lir == 0) stats[row] = rstd;
    }
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = lir + i * TPR;
      if (rv && c < nvec) {
        float g[8], o[8];
        unpack8(gamma[c], g);
        if (kLayer) {
          float bt[8];
          unpack8(beta[c], bt);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = (xv[i][j] - mean) * rstd * g[j] + bt[j];
        } else {
          // norms.py:45-52: normalise in fp32, cast to the 16-bit dtype, THEN multiply by scale (16-bit product)
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = round_bf16(xv[i][j] * rstd) * g[j];
        }
        y[base + c] = pack8(o);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward. dx = rstd * (g - xhat * mean(g*xhat) [- mean(g)])  with g = dy * gamma;  partial dgamma/dbeta per CTA.
// ------------------------------------------------------------------------------------------------------------
template <bool kLayer, int TPR, int VPT, bool kDrop>
__global__ void __launch_bounds__(NORM_THREADS) norm_bwd_kernel(
    const uint4* __restrict__ dy, const uint4* __restrict__ x, const uint4* __restrict__ gamma,
    const float* __restrict__ stats, const uint4* __restrict__ dres, uint4* __restrict__ dx,
    float* __restrict__ partial /* [grid, (kLayer?2:1) * cols] */, int rows, int cols, uint4* __restrict__ dbranch,
    const DropArgs drop) {
  constexpr int RPC = NORM_THREADS / TPR;
  __shared__ float red[RPC * 2 * (TPR / 32)];
  extern __shared__ float comb[];  // [RPC][width] when RPC > 1
  const int nvec = cols >> 3;
  const int row_slot = threadIdx.x / TPR, lir = threadIdx.x % TPR;
  const int width = cols * (kLayer ? 2 : 1);
  float dg[VPT][8], db[kLayer ? VPT : 1][8];
  uint32_t s_lo, s_hi;
  drop_stream<kDrop>(drop.stream_base, drop.site, s_lo, s_hi);
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) { dg[i][j] = 0.f; if (kLayer) db[i][j] = 0.f; }

  for (int base_row = blockIdx.x * RPC; base_row < rows; base_row += gridDim.x * RPC) {
    const int row = base_row + row_slot;
    const bool rv = row < rows;
    const size_t base = size_t(row) * nvec;
    const float mean = (kLayer && rv) ? stats[2 * row] : 0.f;
    const float rstd = rv ? (kLayer ? stats[2 * row + 1] : stats[row]) : 0.f;
    float xh[VPT][8], g[VPT][8];
    uint4 rq[VPT];   // residual-branch gradient, fetched WITH x / dy (one memory round trip per row instead of two)
    float s_g = 0.f, s_gx = 0.f;
    // keep bits of the row's vectors (8 per vector), drawn while the fewest values are live; applied to dbranch at the end
    uint64_t keep = 0;
    if constexpr (kDrop) {
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int c = lir + i * TPR;
        if (rv && c < nvec) keep |= uint64_t(keep_bits8(drop.seed, s_lo, s_hi, drop.thr, row, c)) << (8 * i);
      }
    }
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = lir + i * TPR;
      rq[i] = (dres != nullptr && rv && c < nvec) ? dres[base + c] : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = lir + i * TPR;
      if (rv && c < nvec) {
        float xv[8], dyv[8], gm[8];
        unpack8(x[base + c], xv);
        unpack8(dy[base + c], dyv);
        unpack8(gamma[c], gm);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] = (xv[j] - mean) * rstd;
          g[i][j] = dyv[j] * gm[j];
          s_g += g[i][j];
          s_gx += g[i][j] * xh[i][j];
          dg[i][j] += dyv[j] * (kLayer ? xh[i][j] : round_bf16(xh[i][j]));
          if (kLayer) db[i][j] += dyv[j];
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) { xh[i][j] = 0.f; g[i][j] = 0.f; }
      }
    }
    row_sum2<TPR>(s_g, s_gx, red, row_slot, lir);
    const float m_g = kLayer ? s_g / cols : 0.f;
    const float m_gx = s_gx / cols;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = lir + i * TPR;
      if (rv && c < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (g[i][j] - m_g - xh[i][j] * m_gx);
        {
          float r[8];
          unpack8(rq[i], r);   // zeros when there is no residual branch
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        dx[base + c] = pack8(o);
        if constexpr (kDrop) {
          apply_keep8(uint32_t(keep >> (8 * i)) & 0xffu, drop.keep_scale, o);
          dbranch[base + c] = pack8(o);
        }
      }
    }
  }
  // combine the CTA's row slots in a fixed order, then write this CTA's partial weight gradients
  float* pg = partial + size_t(blockIdx.x) * width;
  if (RPC == 1) {
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = lir + i * TPR;
      if (c < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          pg[c * 8 + j] = dg[i][j];
          if (kLayer) pg[cols + c * 8 + j] = db[i][j];
        }
      }
    }
  } else {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = lir + i * TPR;
      if (c < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          comb[row_slot * width + c * 8 + j] = dg[i][j];
          if (kLayer) comb[row_slot * width + cols + c * 8 + j] = db[i][j];
        }
      }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < width; c += NORM_THREADS) {
      float t = 0.f;
#pragma unroll
      for (int r = 0; r < RPC; ++r) t += comb[r * width + c];
      pg[c] = t;
    }
  }
}

// Column-wise reduction of partial[nparts, width] (fp32). Columns [0, split) go to out0, [split, width) to out1.
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ partial, void* __restrict__ out0,
                                                     void* __restrict__ out1, int nparts, int width, int split,
                                                     int out_f32, int accumulate) {
  __shared__ float sm[8][33];  // 32 columns x 8 row-lanes
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  float s = 0.f;
  if (col < width) {
    // fixed summation order (deterministic), eight independent loads in flight per thread: the chain of dependent
    // L2 round trips, not bandwidth, is what this stage costs
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int r = rl;
    for (; r + 56 < nparts; r += 64) {
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] += partial[size_t(r + 8 * u) * width + col];
    }
    for (int u = 0; r < nparts; r += 8, ++u) a[u] += partial[size_t(r) * width + col];
    s = ((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7]));
  }
  sm[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && col < width) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x & 31];
    void* out = col < split ? out0 : out1;
    const int c = col < split ? col : col - split;
    if (out_f32) {
      float* o = reinterpret_cast<float*>(out);
      o[c] = accumulate ? o[c] + t : t;
    } else {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
      o[c] = __float2bfloat16(accumulate ? __bfloat162float(o[c]) + t : t);
    }
  }
}

// threads per row: smallest of {32,64,128,256} that keeps <= 4 vectors per thread (more only for cols > 8192)
static void norm_shape(int64_t cols, int& tpr, int& vpt) {
  const int nvec = int(cols / 8);
  tpr = 32;
  while (tpr < 256 && (nvec + tpr - 1) / tpr > 4) tpr *= 2;
  vpt = (nvec + tpr - 1) / tpr;
}
// backward: the thread also carries fp32 weight-gradient partials for every column it owns, so at most 3 vectors per thread
// (with 4: 162 registers, ONE resident CTA per SM, 1.5 TB/s on 16384 x 2048 — rows in flight, not bandwidth, bound it;
// with 2-3: 80-123 registers, 2-3 CTAs per SM, 2.5 TB/s)
static void norm_shape_bwd(int64_t cols, int& tpr, int& vpt) {
  const int nvec = int(cols / 8);
  tpr = 32;
  while (tpr < 256 && (nvec + tpr - 1) / tpr > 3) tpr *= 2;
  vpt = (nvec + tpr - 1) / tpr;
}
static int norm_grid(int64_t rows, int tpr) {
  const int rpc = NORM_THREADS / tpr;
  const int64_t groups = (rows + rpc - 1) / rpc;
  static const int mult = [] { const char* e = getenv("FSB_NORM_GRID_MULT"); return e ? atoi(e) : 4; }();   // CTAs per SM (tuning knob)
  const int64_t cap = int64_t(mult) * num_sms();
  return int(groups < cap ? groups : cap);
}

#define FSB_NORM_DISPATCH(KERNEL_LAUNCH)                                                                      \
  switch (tpr) {                                                                                               \
    case 32:  switch (vpt) { case 1: KERNEL_LAUNCH(32, 1); break; case 2: KERNEL_LAUNCH(32, 2); break;         \
                             case 3: KERNEL_LAUNCH(32, 3); break; default: KERNEL_LAUNCH(32, 4); break; } break; \
    case 64:  switch (vpt) { case 1: KERNEL_LAUNCH(64, 1); break; case 2: KERNEL_LAUNCH(64, 2); break;         \
                             case 3: KERNEL_LAUNCH(64, 3); break; default: KERNEL_LAUNCH(64, 4); break; } break; \
    case 128: switch (vpt) { case 1: KERNEL_LAUNCH(128, 1); break; case 2: KERNEL_LAUNCH(128, 2); break;       \
                             case 3: KERNEL_LAUNCH(128, 3); break; default: KERNEL_LAUNCH(128, 4); break; } break; \
    default:  switch (vpt) { case 1: KERNEL_LAUNCH(256, 1); break; case 2: KERNEL_LAUNCH(256, 2); break;        \
                             case 3: KERNEL_LAUNCH(256, 3); break; case 4: KERNEL_LAUNCH(256, 4); break;        \
                             case 5: KERNEL_LAUNCH(256, 5); break; case 6: KERNEL_LAUNCH(256, 6); break;        \
                             case 7: KERNEL_LAUNCH(256, 7); break; default: KERNEL_LAUNCH(256, 8); break; } break; \
  }

template <bool kLayer, bool kDrop = false>
static int norm_fwd(const void* x, const void* residual, const void* gamma, const void* beta, void* y, void* sum_out,
                    float* stats, int64_t rows, int64_t cols, float eps, cudaStream_t st, const DropArgs& drop = DropArgs{}) {
  FSB_REQUIRE(rows > 0 && cols > 0 && cols % 8 == 0 && cols <= 16384 && rows < (1 << 30),
              "norm_fwd: bad shape rows=%ld cols=%ld", (long)rows, (long)cols);
  FSB_REQUIRE(x && gamma && y && stats && (!kLayer || beta), "norm_fwd: null pointer");
  FSB_REQUIRE(residual == nullptr || sum_out != nullptr, "norm_fwd: residual given without sum_out");
  FSB_REQUIRE(aligned16(x) && aligned16(y) && aligned16(gamma) && aligned16(residual) && aligned16(sum_out) &&
                  aligned16(beta),
              "norm_fwd: pointers must be 16-byte aligned");
  int tpr, vpt;
  norm_shape(cols, tpr, vpt);
  const int grid = norm_grid(rows, tpr);
#define L(T, V)                                                                                                   \
  if constexpr (!kDrop || V <= NORM_DROP_MAX_VPT)                                                                  \
  norm_fwd_kernel<kLayer, T, V, kDrop><<<grid, NORM_THREADS, 0, st>>>(                                             \
      (const uint4*)x, (const uint4*)residual, (const uint4*)gamma, (const uint4*)beta, (uint4*)y, (uint4*)sum_out, stats, \
      int(rows), int(cols), eps, drop)
  FSB_NORM_DISPATCH(L)
#undef L
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

template <bool kLayer, int T, int V, bool kDrop>
static cudaError_t norm_bwd_smem_attr(size_t bytes) {
  static size_t configured = 0;
  if (bytes > configured) {
    // the dynamic bytes and the kernel's static shared memory together may not pass 48 KiB without the opt-in (LayerNorm at
    // 3072 columns asks for exactly 48 KiB of dynamic memory)
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, norm_bwd_kernel<kLayer, T, V, kDrop>);
    if (e != cudaSuccess) return e;
    if (bytes + fa.sharedSizeBytes > 48 * 1024) {
      e = cudaFuncSetAttribute(norm_bwd_kernel<kLayer, T, V, kDrop>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes));
      if (e != cudaSuccess) return e;
    }
    configured = bytes;
  }
  return cudaSuccess;
}

template <bool kLayer, bool kDrop = false>
static int norm_bwd(const void* dy, const void* x, const void* gamma, const float* stats, const void* dres, void* dx,
                    void* dgamma, void* dbeta, int wgrad_dtype, int accumulate, void* workspace, size_t ws_bytes,
                    int64_t rows, int64_t cols, cudaStream_t st, void* dbranch = nullptr, const DropArgs& drop = DropArgs{}) {
  FSB_REQUIRE(rows > 0 && cols > 0 && cols % 8 == 0 && cols <= 16384 && rows < (1 << 30),
              "norm_bwd: bad shape rows=%ld cols=%ld", (long)rows, (long)cols);
  FSB_REQUIRE(dy && x && gamma && stats && dx && dgamma && workspace && (!kLayer || dbeta), "norm_bwd: null pointer");
  FSB_REQUIRE(aligned16(dy) && aligned16(x) && aligned16(gamma) && aligned16(dres) && aligned16(dx),
              "norm_bwd: pointers must be 16-byte aligned");
  int tpr, vpt;
  norm_shape_bwd(cols, tpr, vpt);
  const int grid = norm_grid(rows, tpr);
  const int width = int(cols) * (kLayer ? 2 : 1);
  const size_t need = size_t(grid) * width * sizeof(float);
  FSB_REQUIRE(ws_bytes >= need, "norm_bwd: workspace %zu < %zu bytes", ws_bytes, need);
  const int rpc = NORM_THREADS / tpr;
  const size_t smem = rpc > 1 ? size_t(rpc) * width * sizeof(float) : 0;
  cudaError_t e = cudaSuccess;
#define L(T, V)                                                                                                    \
  if constexpr (!kDrop || V <= NORM_DROP_MAX_VPT) {                                                                \
    e = norm_bwd_smem_attr<kLayer, T, V, kDrop>(smem);                                                             \
    if (e == cudaSuccess)                                                                                          \
      norm_bwd_kernel<kLayer, T, V, kDrop><<<grid, NORM_THREADS, smem, st>>>(                                      \
          (const uint4*)dy, (const uint4*)x, (const uint4*)gamma, stats, (const uint4*)dres, (uint4*)dx,               \
          (float*)workspace, int(rows), int(cols), (uint4*)dbranch, drop);                                         \
  }
  FSB_NORM_DISPATCH(L)
#undef L
  if (e != cudaSuccess) {
    set_error("norm_bwd: cudaFuncSetAttribute(%zu B) failed: %s", smem, cudaGetErrorString(e));
    return FSB_ERR_CUDA;
  }
  FSB_CUDA_LAUNCH_CHECK();
  colsum_kernel<<<(width + 31) / 32, 256, 0, st>>>((const float*)workspace, dgamma, dbeta, grid, width, int(cols),
                                                   wgrad_dtype == FSB_F32, accumulate);
  FSB_CUDA_LAUNCH_CHECK();
  return FSB_OK;
}

}  // namespace fsb

using namespace fsb;

extern "C" size_t fsb_norm_bwd_workspace_bytes(int64_t rows, int64_t cols, int is_layernorm) {
  int tpr, vpt;
  norm_shape_bwd(cols, tpr, vpt);
  return size_t(norm_grid(rows, tpr)) * size_t(cols) * (is_layernorm ? 2 : 1) * sizeof(float);
}
extern "C" int fsb_rmsnorm_fwd(const void* x, const void* residual, const void* scale, void* y, void* sum_out,
                               float* rstd, int64_t rows, int64_t cols, float eps, fsb_stream_t st) {
  return norm_fwd<false>(x, residual, scale, nullptr, y, sum_out, rstd, rows, cols, eps, (cudaStream_t)st);
}
extern "C" int fsb_rmsnorm_bwd(const void* dy, const void* x, const void* scale, const float* rstd, const void* dres,
                               void* dx, void* dscale, int wgrad_dtype, int accumulate, void* workspace,
                               size_t workspace_bytes, int64_t rows, int64_t cols, fsb_stream_t st) {
  return norm_bwd<false>(dy, x, scale, rstd, dres, dx, dscale, nullptr, wgrad_dtype, accumulate, workspace,
                         workspace_bytes, rows, cols, (cudaStream_t)st);
}
extern "C" int fsb_layernorm_fwd(const void* x, const void* residual, const void* gamma, const void* beta, void* y,
                                 void* sum_out, float* mean_rstd, int64_t rows, int64_t cols, float eps,
                                 fsb_stream_t st) {
  return norm_fwd<true>(x, residual, gamma, beta, y, sum_out, mean_rstd, rows, cols, eps, (cudaStream_t)st);
}
extern "C" int fsb_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean_rstd,
                                 const void* dres, void* dx, void* dgamma, void* dbeta, int wgrad_dtype,
                                 int accumulate, void* workspace, size_t workspace_bytes, int64_t rows, int64_t cols,
                                 fsb_stream_t st) {
  return norm_bwd<true>(dy, x, gamma, mean_rstd, dres, dx, dgamma, dbeta, wgrad_dtype, accumulate, workspace,
                        workspace_bytes, rows, cols, (cudaStream_t)st);
}
extern "C" int fsb_layernorm_fwd_dropout(const void* x, const void* residual, const void* gamma, const void* beta, void* y,
                                         void* sum_out, float* mean_rstd, int64_t rows, int64_t cols, float eps, float p,
                                         uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  if (p == 0.f) return norm_fwd<true>(x, residual, gamma, beta, y, sum_out, mean_rstd, rows, cols, eps, (cudaStream_t)st);
  FSB_REQUIRE(residual != nullptr, "layernorm_fwd_dropout: the dropped branch needs a residual");
  FSB_REQUIRE(cols <= 8 * 256 * NORM_DROP_MAX_VPT, "layernorm_fwd_dropout: cols %ld > %d with p > 0", (long)cols,
              8 * 256 * NORM_DROP_MAX_VPT);
  return norm_fwd<true, true>(x, residual, gamma, beta, y, sum_out, mean_rstd, rows, cols, eps, (cudaStream_t)st, d);
}
extern "C" int fsb_layernorm_bwd_dropout(const void* dy, const void* x, const void* gamma, const float* mean_rstd,
                                         const void* dres, void* dx, void* dbranch, void* dgamma, void* dbeta,
                                         int wgrad_dtype, int accumulate, void* workspace, size_t workspace_bytes,
                                         int64_t rows, int64_t cols, float p, uint64_t seed, const int64_t* stream_base,
                                         int64_t site, fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  FSB_REQUIRE(dbranch != nullptr && aligned16(dbranch), "layernorm_bwd_dropout: dbranch must be a 16-byte aligned buffer");
  if (p == 0.f) {   // no mask: the branch gradient is the gradient of the sum
    if (int rc = norm_bwd<true>(dy, x, gamma, mean_rstd, dres, dx, dgamma, dbeta, wgrad_dtype, accumulate, workspace,
                                workspace_bytes, rows, cols, (cudaStream_t)st))
      return rc;
    cudaError_t e = cudaMemcpyAsync(dbranch, dx, size_t(rows) * size_t(cols) * 2, cudaMemcpyDeviceToDevice, (cudaStream_t)st);
    if (e != cudaSuccess) {
      set_error("layernorm_bwd_dropout: copy of dx failed: %s", cudaGetErrorString(e));
      return FSB_ERR_CUDA;
    }
    return FSB_OK;
  }
  FSB_REQUIRE(cols <= 8 * 256 * NORM_DROP_MAX_VPT, "layernorm_bwd_dropout: cols %ld > %d with p > 0", (long)cols,
              8 * 256 * NORM_DROP_MAX_VPT);
  return norm_bwd<true, true>(dy, x, gamma, mean_rstd, dres, dx, dgamma, dbeta, wgrad_dtype, accumulate, workspace,
                              workspace_bytes, rows, cols, (cudaStream_t)st, dbranch, d);
}
extern "C" int fsb_rmsnorm_fwd_dropout(const void* x, const void* residual, const void* scale, void* y, void* sum_out,
                                       float* rstd, int64_t rows, int64_t cols, float eps, float p, uint64_t seed,
                                       const int64_t* stream_base, int64_t site, fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  if (p == 0.f) return norm_fwd<false>(x, residual, scale, nullptr, y, sum_out, rstd, rows, cols, eps, (cudaStream_t)st);
  FSB_REQUIRE(residual != nullptr, "rmsnorm_fwd_dropout: the dropped branch needs a residual");
  FSB_REQUIRE(cols <= 8 * 256 * NORM_DROP_MAX_VPT, "rmsnorm_fwd_dropout: cols %ld > %d with p > 0", (long)cols,
              8 * 256 * NORM_DROP_MAX_VPT);
  return norm_fwd<false, true>(x, residual, scale, nullptr, y, sum_out, rstd, rows, cols, eps, (cudaStream_t)st, d);
}
extern "C" int fsb_rmsnorm_bwd_dropout(const void* dy, const void* x, const void* scale, const float* rstd, const void* dres,
                                       void* dx, void* dbranch, void* dscale, int wgrad_dtype, int accumulate, void* workspace,
                                       size_t workspace_bytes, int64_t rows, int64_t cols, float p, uint64_t seed,
                                       const int64_t* stream_base, int64_t site, fsb_stream_t st) {
  DropArgs d;
  if (int rc = make_drop_args(p, seed, stream_base, site, &d)) return rc;
  FSB_REQUIRE(dbranch != nullptr && aligned16(dbranch), "rmsnorm_bwd_dropout: dbranch must be a 16-byte aligned buffer");
  if (p == 0.f) {   // no mask: the branch gradient is the gradient of the sum
    if (int rc = norm_bwd<false>(dy, x, scale, rstd, dres, dx, dscale, nullptr, wgrad_dtype, accumulate, workspace,
                                 workspace_bytes, rows, cols, (cudaStream_t)st))
      return rc;
    cudaError_t e = cudaMemcpyAsync(dbranch, dx, size_t(rows) * size_t(cols) * 2, cudaMemcpyDeviceToDevice, (cudaStream_t)st);
    if (e != cudaSuccess) {
      set_error("rmsnorm_bwd_dropout: copy of dx failed: %s", cudaGetErrorString(e));
      return FSB_ERR_CUDA;
    }
    return FSB_OK;
  }
  FSB_REQUIRE(cols <= 8 * 256 * NORM_DROP_MAX_VPT, "rmsnorm_bwd_dropout: cols %ld > %d with p > 0", (long)cols,
              8 * 256 * NORM_DROP_MAX_VPT);
  return norm_bwd<false, true>(dy, x, scale, rstd, dres, dx, dscale, nullptr, wgrad_dtype, accumulate, workspace,
                               workspace_bytes, rows, cols, (cudaStream_t)st, dbranch, d);
}
