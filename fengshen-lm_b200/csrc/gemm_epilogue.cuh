// fsb200 — the GELU forms of the GEMM epilogues (gemm.cu, gemm_fp8.cu). Both GEMMs evaluate FSB_EPI_GELU_TANH /
// FSB_EPI_GELU_ERF with this device code, so the same fp32 pre-activation gives the same bits whichever GEMM produced it.
// (The standalone activation kernels in elementwise.cu keep their own, libm-based forms.)
#pragma once
#include "ptx.cuh"

namespace fsb {

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

}  // namespace fsb
