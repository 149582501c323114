// esm_b200 — Gibbs sampling of protein sequences and MSA Transformer alignments (esm_b200/sampling.py), the
// definitions in include/esmb200.h at esmb200_sample_order / esmb200_sample_rows.
//
// Random stream: R(c0, c1, c2, c3) = Philox4x32-10 (the toolkit's curand_Philox4x32_10) with counter (c0, c1, c2, c3)
// and key (seed mod 2^32, seed >> 32). No state is carried between launches: every draw is a pure function of
// (seed, chain, step, entry), so the result does not depend on how chains are batched.
//   sample_order_kernel  the sort keys R(sweep, chain, p, 0).x * 2^20 + p of one sweep's visiting order
//   sample_rows_kernel   one warp per resampled entry: tempered logits of a token set of 1 ... 32 ids, Gumbel-max
//                        draw with the uniforms of R(step, chain, p, 1 + a / 4), the token written in place, its log q
//   sample_logp_kernel   per chain, the block's log q summed in block order
#pragma once

#include <cuda_runtime.h>
#include <curand_philox4x32_x.h>
#include <stdint.h>

#include "elementwise.cuh"

namespace esmb200 {

__device__ __forceinline__ uint4 sample_philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint64_t seed) {
  return curand_Philox4x32_10(make_uint4(c0, c1, c2, c3), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
}

// u = ((r >> 8) + 0.5) * 2^-24, rounded toward zero to fp32 in one step. Below 1/2 the value is exact. Above it needs
// 25 significant bits; rounding to nearest would take the largest word to 1.0, whose Gumbel noise is +inf, while
// rounding toward zero drops the half and keeps every u in (0, 1).
__device__ __forceinline__ float sample_uniform(uint32_t r) { return __fmaf_rz((float)(r >> 8), 0x1p-24f, 0x1p-25f); }

// keys[c, j] = R(sweep, chain0 + c, p, 0).x * 2^20 + p for p = entries[j] (p < 2^20, so keys never tie).
// Grid-stride over the n_chains * n keys.
__global__ void __launch_bounds__(256)
sample_order_kernel(const int64_t* __restrict__ entries, int n, int64_t total, uint32_t chain0, uint32_t sweep,
                    uint64_t seed, int64_t* __restrict__ keys) {
  for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (int64_t)gridDim.x * 256) {
    const int64_t c = e / n;
    const int64_t p = entries[e - c * n];
    const uint4 r = sample_philox(sweep, chain0 + (uint32_t)c, (uint32_t)p, 0u, seed);
    keys[e] = ((int64_t)r.x << 20) + p;
  }
}

// One warp per row r (8 per block, any number of rows along grid x): chain chain0 + r / per_chain, entry
// p = entries[r] of an alignment of R rows and C columns whose column 0 is <cls> (a protein is R = 1, C = T - 1).
// Lane a < n_set holds z_a = logits[r, token_set[a]] / tau (an IEEE division, -INFINITY on the other lanes) and scores
// z_a - logf(-logf(u_a)), u_a from word a mod 4 of R(step, chain, p, 1 + a / 4); the xor-butterfly keeps the larger
// score and, on a tie, the smaller a. token_set[a*] goes to tokens[c * chain_stride + (p / (C - 1)) * C + 1 +
// p % (C - 1)], and log q = (z_a* - m) - lse from warp_row_lse is log_softmax_rows_kernel's value for target a*. An
// entry outside [0, R (C - 1)) writes no token and a NaN log q.
__global__ void __launch_bounds__(256)
sample_rows_kernel(const float* __restrict__ logits, int64_t ld, int64_t n, const int* __restrict__ token_set,
                   int n_set, float tau, uint64_t seed, uint32_t step, uint32_t chain0, int per_chain,
                   const int64_t* __restrict__ entries, int64_t* __restrict__ tokens, int64_t chain_stride, int R,
                   int C, float* __restrict__ logq) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= n) return;
  const int64_t c = row / per_chain;
  const int64_t p = entries[row];
  const int tok = lane < n_set ? token_set[lane] : 0;
  const float z = lane < n_set ? logits[row * ld + tok] / tau : -INFINITY;
  float m, lse;
  warp_row_lse(z, -INFINITY, m, lse);
  float score = -INFINITY;
  if (lane < n_set) {
    const uint4 r = sample_philox(step, chain0 + (uint32_t)c, (uint32_t)p, 1u + (uint32_t)lane / 4, seed);
    const int w = lane & 3;
    const uint32_t word = w == 0 ? r.x : w == 1 ? r.y : w == 2 ? r.z : r.w;
    score = z + -logf(-logf(sample_uniform(word)));
  }
  int best = lane;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float s2 = __shfl_xor_sync(0xffffffffu, score, o);
    const int b2 = __shfl_xor_sync(0xffffffffu, best, o);
    if (s2 > score || (s2 == score && b2 < best)) {
      score = s2;
      best = b2;
    }
  }
  best = __shfl_sync(0xffffffffu, best, 0);
  const float zb = __shfl_sync(0xffffffffu, z, best);
  const int drawn = __shfl_sync(0xffffffffu, tok, best);
  if (lane == 0) {
    const int64_t W = C - 1;
    if (p >= 0 && p < (int64_t)R * W) {
      tokens[c * chain_stride + (p / W) * C + 1 + p % W] = drawn;
      logq[row] = (zb - m) - lse;
    } else {
      logq[row] = __int_as_float(0x7fc00000);
    }
  }
}

// logp[c * stride] = the per_chain values logq[c * per_chain + j] summed in j order from +0 (fp32).
__global__ void __launch_bounds__(256)
sample_logp_kernel(const float* __restrict__ logq, int64_t n_chains, int per_chain, float* __restrict__ logp,
                   int64_t stride) {
  const int64_t c = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (c >= n_chains) return;
  float acc = 0.f;
  for (int j = 0; j < per_chain; ++j) acc += logq[c * per_chain + j];
  logp[c * stride] = acc;
}

}  // namespace esmb200
