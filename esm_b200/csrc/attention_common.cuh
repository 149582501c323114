// esm_b200 — definitions shared by the attention kernels (sm_90a, head_dim 64 per column slot): parameter block and
// the warp-level Q.K^T tile product.
//
// The kernels replace esm/multihead_attention.py:357-394 (bmm(q,k^T) -> key-padding -inf mask -> fp32 softmax ->
// bmm(P,v) -> (T,B,E) merge) without ever writing S or P to HBM.  Inputs come from the QKV GEMM epilogue: qkv fp16
// [B*T, 3E], q already scaled by d^-1/2 and rotated, k rotated.
#pragma once

#include "common.cuh"

namespace esmb200 {

struct AttnParams {
  int B, T, H, E;           // E = H * 64 * slots: width of q, of k, of v and of ctx
  const uint32_t* keybits;  // [B, words]: bit i of word w set <=> key 32*w+i is attendable (not pad, < T)
  const int* kvlen;         // [B]: 1 + index of the last attendable key (0 if none)
  int words;                // words per sequence, multiple of 4
  __half* ctx;              // [B*T, E] attention output, heads merged (column h*64 + j)
  float* row_max;           // optional [B,H,T]: final softmax row max (of the scaled scores) ...
  float* row_sum;           // optional [B,H,T]: ... and row sum of exp(s - max), for the probability kernels
  int lo_off = 0;           // fp32x3 precision: column offset (elements) of the lo halves in qkv [M, 6E] (= 3E)
  int slots = 1;            // 64-wide column slots per head: 1 (head_dim <= 64) or 2 (head_dim <= 128); E = H * 64 * slots
  int cols = 1;             // sequence s = (s / cols, s % cols) of a [B/cols, T, cols, 3E] tensor (fp32x3: 6E)
                            // (MSA column attention: the T tokens of a sequence are `cols` rows apart)
};

namespace attn_cfg {
constexpr int HEAD_DIM = 64;
constexpr int TILE_BYTES = 128 * 64 * 2;  // 16 KB: 128 rows x 128 bytes
constexpr float LOG2E = 1.4426950408889634f;
}  // namespace attn_cfg

// s[NB][4] += Q[16 rows from q_row0] . K[NB*8 keys from k_row0]^T over 64 head columns: Q and K are SW128 tiles with
// 128-byte rows (TMA boxes of 64 fp16 columns).  Fragment layout of s: see mma16816 (row g / g + 8, key 8 nb + 2c..).
template <int NB>
__device__ __forceinline__ void qk_tile(float (&s)[NB][4], uint32_t q_base, uint32_t q_row0, uint32_t k_base,
                                        uint32_t k_row0) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[4];
    ldsm_a(q_base, q_row0, kk, a);
#pragma unroll
    for (int n2 = 0; n2 < NB / 2; ++n2) {
      uint32_t b[4];
      ldsm_b(k_base, k_row0 + 16 * n2, kk, b);
      mma16816(s[2 * n2], a, b[0], b[1]);
      mma16816(s[2 * n2 + 1], a, b[2], b[3]);
    }
  }
}

// normalised probability of score s: exp(s - m) * inv for an attendable key (bit key % 32 of its key word), else 0
__device__ __forceinline__ float masked_prob(float s, uint32_t kw, int key, float mneg, float inv) {
  constexpr float LOG2E = attn_cfg::LOG2E;
  return ((kw >> (key & 31)) & 1u) ? ex2_approx(fmaf(s, LOG2E, mneg)) * inv : 0.f;
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

}  // namespace esmb200
