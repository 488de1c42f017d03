// fsb200 — host-side helpers shared by every translation unit of libfsb200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/fsb200.h"

namespace fsb {

// Thread-local error string returned by fsb_last_error().
void set_error(const char* fmt, ...);

#define FSB_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      ::fsb::set_error(__VA_ARGS__);      \
      return FSB_ERR_INVALID;             \
    }                                     \
  } while (0)

#define FSB_CUDA_LAUNCH_CHECK()                                                       \
  do {                                                                                \
    cudaError_t e__ = cudaGetLastError();                                             \
    if (e__ != cudaSuccess) {                                                         \
      ::fsb::set_error("%s:%d CUDA launch error: %s", __FILE__, __LINE__,             \
                       cudaGetErrorString(e__));                                      \
      return FSB_ERR_CUDA;                                                            \
    }                                                                                 \
  } while (0)

int num_sms();

// SMs left to concurrently running communication kernels (fsb_set_reserved_sms): a persistent GEMM CTA fills an SM
// (all of its registers), so a collective that overlaps backward would otherwise push GEMM CTAs into a second wave.
// Every persistent GEMM (gemm.cu, gemm_fp8.cu) sizes its grid with gemm_sms().
extern int g_reserved_sms;
static inline int gemm_sms() {
  const int n = num_sms() - g_reserved_sms;
  return n < 1 ? 1 : n;
}

// 2-D / 3-D bf16 / fp32 tensor map with 128B swizzle. dims/box innermost-first; strides (bytes) for dims 1.. .
// Returns 0 on success (error string set otherwise).
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);
int make_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box);
int make_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box);
// bf16 map over a packed attention activation buffer: dims {width, seq, batch} with rows row_stride elements apart; box
// {64, box_rows, 1}
int make_attn_tmap(CUtensorMap* tm, const void* base, int64_t row_stride, int64_t width, int64_t seq, int64_t batch,
                   int box_rows);
// Segment mode (kSeg) of the attention forward / backward kernels for packed rows (the segment forms of fsb_sdpa_fwd /
// fsb_sdpa_bwd): none, causal inside each segment, bidirectional inside each segment, or cross-attention from each query's
// segment to its key range in another sequence
enum AttnSegMode : int { kSegNone = 0, kSegCausal = 1, kSegBidir = 2, kSegCross = 3 };

// The kernel instantiation (D, kBias, kDropout, kSeg) one attention call runs; key() is what the launchers switch over.
struct AttnForm {
  int d;
  bool bias, dropout;
  AttnSegMode seg;
  constexpr int key() const { return d << 8 | int(bias) << 4 | int(dropout) << 3 | int(seg); }
};
// The table of forms of include/fsb200.h, shared by fsb_sdpa_fwd and fsb_sdpa_bwd: picks the form from the arguments that
// select it and refuses (FSB_ERR_INVALID, error string prefixed with `what`) every combination no kernel is built for.
int resolve_attn_form(const char* what, int head_dim, int causal, const void* kv_mask, const void* rel_bias,
                      const int32_t* seg_start, const int32_t* seg_end, const int32_t* q_start, const int32_t* q_end,
                      float p, int64_t seq_q, int64_t seq_kv, AttnForm* form);

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Lets kKernel launch with `bytes` of dynamic shared memory (above the 48 KB default); the attribute is set on the first
// successful call only. The kernel is a template argument so that every kernel has its own flag: kernels of one signature
// share a function-pointer type.
template <auto kKernel>
int ensure_smem(int bytes, const char* what) {
  static bool configured = false;
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute(%d B smem) failed: %s", what, bytes, cudaGetErrorString(e));
      return FSB_ERR_CUDA;
    }
    configured = true;
  }
  return FSB_OK;
}

}  // namespace fsb
