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

// ---- epilogue boxes shared by the fp16 (gemm2.cuh) and fp8 (gemm_fp8.cuh) GEMMs.  A thread of an MMA warpgroup holds
// rows r0 and r0 + 8 of the box; `acc` points at the box's accumulators in the wgmma fragment layout,
// acc[4 b + 2 hr + {0, 1}] = row r0 + 8 hr, columns col0 + 8 b + 2 c + {0, 1}.

// An fp16 64 x 64 output box of one MMA warpgroup into a 128B-swizzled staging buffer (the layout the output TMA map
// reads): h[2 b + hr] holds the warp's rows g + 8 hr, columns 8 b + 2 c ..+1 (the accumulator fragment layout, which is
// stmatrix's).  Each x4 writes blocks 2s, 2s + 1 for both row halves; 8 rows x 16 bytes per matrix, conflict-free.
__device__ __forceinline__ void stage_box_f16(uint32_t buf, uint32_t warp, uint32_t lane, const uint32_t (&h)[16]) {
  const uint32_t m = lane / 8;  // matrix this lane addresses: block 2s + m / 2, row half m % 2
#pragma unroll
  for (int s = 0; s < 4; ++s)
    stsm_x4(sw128(buf, warp * 16 + (m % 2) * 8 + lane % 8, 2 * s + m / 2), h[4 * s], h[4 * s + 1], h[4 * s + 2],
            h[4 * s + 3]);
}

// EPI_QKV_ROPE, one 64-column box (32 accumulators): + bias, q columns * q_scale, rotate-half RoPE on q and k (column j
// pairs with j + 32, same thread) -> fp16 pairs hi[2 b + hr]; SPLIT also the lo halves rn(y - hi).
template <bool SPLIT>
__device__ __forceinline__ void epi_qkv_box(const float* acc, const GemmParams& p, int col0, int r0, uint32_t c,
                                            uint32_t (&hi)[16], uint32_t (&lo)[16]) {
  const int sect = col0 / p.E;  // 0 q, 1 k, 2 v
  const float sc = (sect == 0) ? p.q_scale : 1.0f;
  // Every bias / table load of the box is issued before the first is used: one memory latency per box rather
  // than one per column pair (the rotation's branch would otherwise split them into dependent steps).
  float2 bl[4], bh[4], cs[2][4], sn[2][4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    bl[q] = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * q + 2 * (int)c));
    bh[q] = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 32 + 8 * q + 2 * (int)c));
  }
  const bool rotate = sect < 2 && p.rope_cos != nullptr;  // uniform over the box
  if (rotate) {
    const int ld = p.rope_ld == 64 ? 64 : 32;
    const int slot = p.rope_ld == 64 ? ((col0 >> 6) & 1) : 0;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int t = (r0 + 8 * hr) % p.T;  // rows >= M read a valid table row too; TMA drops them
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const size_t at = (size_t)t * ld + slot * 32 + 8 * q + 2 * (int)c;
        cs[hr][q] = __ldg(reinterpret_cast<const float2*>(p.rope_cos + at));
        sn[hr][q] = __ldg(reinterpret_cast<const float2*>(p.rope_sin + at));
      }
    }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {  // column pair (j, j + 1) and (j + 32, j + 33) of the box, j = 8 q + 2 c
      float a0 = (acc[4 * q + 2 * hr] + bl[q].x) * sc;
      float a1 = (acc[4 * q + 2 * hr + 1] + bl[q].y) * sc;
      float b0 = (acc[4 * (q + 4) + 2 * hr] + bh[q].x) * sc;
      float b1 = (acc[4 * (q + 4) + 2 * hr + 1] + bh[q].y) * sc;
      if (rotate) {  // rotary_embedding.py:16-20, rotate_half = cat(-x2, x1)
        const float2 co = cs[hr][q], si = sn[hr][q];
        const float ra0 = a0 * co.x - b0 * si.x, rb0 = b0 * co.x + a0 * si.x;
        const float ra1 = a1 * co.y - b1 * si.y, rb1 = b1 * co.y + a1 * si.y;
        a0 = ra0; b0 = rb0; a1 = ra1; b1 = rb1;
      }
      hi[2 * q + hr] = pack_half2(a0, a1);
      hi[2 * (q + 4) + hr] = pack_half2(b0, b1);
      if constexpr (SPLIT) {
        const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&hi[2 * q + hr]));
        const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(&hi[2 * (q + 4) + hr]));
        lo[2 * q + hr] = pack_half2(a0 - fa.x, a1 - fa.y);
        lo[2 * (q + 4) + hr] = pack_half2(b0 - fb.x, b1 - fb.y);
      }
    }
  }
}


}  // namespace esmb200
