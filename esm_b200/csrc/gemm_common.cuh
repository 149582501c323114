// esm_b200 — definitions shared by the GEMM kernels (sm_90a): epilogue ids, parameter block, erf-GELU.
//
// Epilogues (reference lines they replace, esm/...):
//   QKV_ROPE      multihead_attention.py:258-261 (q/k/v Linear + bias, q *= d^-1/2) + :354-355 /
//                 rotary_embedding.py:11-20 (rotate-half RoPE on q,k) -> fp16 [M,3E]
//   BIAS_RESIDUAL multihead_attention.py:395 + modules.py:134, and modules.py:139-140
//                 (Linear + bias, residual add) -> fp32 residual stream updated in place
//   BIAS_GELU     modules.py:138 + :17-24 (fc1 + exact erf GELU) -> fp16 [M,F]
//   BIAS_F32      plain Linear + bias -> fp32 (LM-head dense, modules.py:308)
#pragma once

#include "common.cuh"

namespace esmb200 {

enum : int { EPI_QKV_ROPE = 0, EPI_BIAS_RESIDUAL = 1, EPI_BIAS_GELU = 2, EPI_BIAS_F32 = 3, EPI_BIAS_GELU_F32 = 4 };

struct GemmParams {
  int M, N, K;
  const float* bias;      // [N] fp32 (the output, fp16 or fp32 row-major [M, N], is the kernel's output tensor map)
  // EPI_QKV_ROPE only
  const float* rope_cos;  // [T, rope_ld] fp32 (angle t * inv_freq[j], j < d/2; further columns are padding)
  const float* rope_sin;
  int rope_ld;            // 0 / 32: head_dim <= 64, one 64-wide slot per head; 64: head_dim <= 128, two slots per head —
                          // the odd 64-column groups take table columns [32,64) (elementwise.cuh head_slot)
  int T;                  // tokens per sequence: position of row r is r % T
  int E;                  // embed dim: columns [0,E) = q, [E,2E) = k, [2E,3E) = v
  float q_scale;          // head_dim^-0.5
  int lo_col_off;         // SPLIT kernels with fp16 output: the lo half of column c is written at column c + lo_col_off
};


// Exact-erf GELU x * 0.5 * (1 + erf(x / sqrt 2)) (esm/modules.py:17-24) with erf from Abramowitz & Stegun 7.1.26
// (|erf error| <= 1.5e-7, far below the fp16 rounding of the stored activation): 15 instructions, 2 MUFU,
// against ~25 for libdevice erff. For x >= 0: x - x*q, for x < 0: x*q with q = 0.5 * poly(t) * exp(-x^2/2),
// t = 1 / (1 + p|x|/sqrt 2).
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float poly = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  poly = fmaf(poly, t, 0.5f * 1.421413741f);
  poly = fmaf(poly, t, 0.5f * -0.284496736f);
  poly = fmaf(poly, t, 0.5f * 0.254829592f);
  poly *= t;
  const float e = ex2_approx(z * (z * -1.4426950408889634f));
  const float q = poly * e;
  return x * (x >= 0.f ? 1.0f - q : q);
}

}  // namespace esmb200
