// esm_b200 — need_head_weights=True: the normalised attention probabilities (sm_90a).
#pragma once

#include "attention_common.cuh"

namespace esmb200 {

// ---------------------------------------------------------------------------------------------------------------
// need_head_weights=True: materialise the normalised probabilities (multihead_attention.py:379,397-400).
// One CTA per (key block, query block, sequence*head), sequences from p.b0: S = Q K^T again on the tensor cores (eight
// warps of 16 query rows x 128 keys), then p = exp(s - rowmax) / rowsum with the row statistics saved by the forward
// kernel, fp32 [B,H,T,T].
// ---------------------------------------------------------------------------------------------------------------
struct ProbsParams {
  int B, T, H, E;
  const uint32_t* keybits;
  const int* kvlen;
  int words;
  const float* row_max;
  const float* row_sum;
  float* probs;  // [B,H,T,T], batch b starting at probs + b * batch_stride (elements)
  long long batch_stride;
  int zero_pad_rows;  // 1: rows of padded query tokens are written as zeros (ESM2.forward's stacked result)
  int lo_off;         // fp32x3 precision: column offset of the lo halves in qkv [M, 6E] (0 = plain fp16 operands)
  int slots = 1;      // 2: head_dim <= 128, a head is two adjacent 64-wide column slots (E = H * 128)
  int cols = 1;       // sequence b = (b / cols, b % cols) of a [B/cols, T, cols, 3E] qkv (fp32x3: 6E), as AttnParams::cols
  int b0 = 0;         // the launch's first sequence: grid z holds (sequence - b0, head) pairs (launch_attention_probs)
};

namespace probs_cfg {
constexpr int NUM_THREADS = 256;
constexpr int BLOCK_Q = 128, BLOCK_KV = 128;
constexpr int smem_bytes(int np) { return 2 * np * attn_cfg::TILE_BYTES + 1024 + 64; }
constexpr int MAX_GRID_Z = 65535;
// sequences per launch: grid z holds one index per (sequence, head) pair
inline int seqs_per_launch(int H) { return MAX_GRID_Z / H; }
}  // namespace probs_cfg

// MODE 0: fp16 operands, head_dim <= 64 | 1 (SPLIT): fp32x3 hi|lo operands | 2: two 64-wide slots per head
template <int MODE>
__global__ void __launch_bounds__(probs_cfg::NUM_THREADS, MODE ? 1 : 2)
attention_probs_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const ProbsParams p) {
  using namespace attn_cfg;
  using namespace probs_cfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int NP = MODE ? 2 : 1;
  uint8_t* smem_q = smem;                    // [hi | lo] or [slot 0 | slot 1]
  uint8_t* smem_k = smem + NP * TILE_BYTES;  // [hi | lo] or [slot 0 | slot 1]
  uint64_t* ld_full = reinterpret_cast<uint64_t*>(smem + 2 * NP * TILE_BYTES);

  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = lane / 4, c = lane % 4;
  const int kb = blockIdx.x, qb = blockIdx.y;
  const int b = p.b0 + (int)(blockIdx.z / p.H), h = blockIdx.z % p.H;
  const int q0 = qb * BLOCK_Q, k0 = kb * BLOCK_KV;
  const int row_base = (b / p.cols) * p.T;
  const int x0 = (b % p.cols) * (MODE == 1 ? 6 : 3) * p.E;  // MODE 1: a token's qkv is 6E wide (hi | lo)

  if (threadIdx.x == 0) {
    mbar_init(ld_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  const bool live = k0 < p.kvlen[b];  // otherwise every key of this block is masked: probabilities are exactly 0

  float s[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
  if (live) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(ld_full, 2 * NP * TILE_BYTES);
      const int hc = x0 + h * HEAD_DIM * (MODE == 2 ? 2 : 1), po = MODE == 2 ? HEAD_DIM : p.lo_off;
#pragma unroll
      for (int part = 0; part < NP; ++part) {
        tma_load_2d(smem_q + part * TILE_BYTES, &tmap_qkv, ld_full, hc + part * po, row_base + q0);
        tma_load_2d(smem_k + part * TILE_BYTES, &tmap_qkv, ld_full, p.E + hc + part * po, row_base + k0);
      }
    }
    mbar_wait(ld_full, 0);
    const uint32_t qs = smem_u32(smem_q), ks = smem_u32(smem_k);
    qk_tile<16>(s, qs, warp * 16, ks, 0);
    if constexpr (MODE == 1) {  // + q_lo k_hi + q_hi k_lo
      qk_tile<16>(s, qs + TILE_BYTES, warp * 16, ks, 0);
      qk_tile<16>(s, qs, warp * 16, ks + TILE_BYTES, 0);
    }
    if constexpr (MODE == 2) qk_tile<16>(s, qs + TILE_BYTES, warp * 16, ks + TILE_BYTES, 0);  // + q[slot 1] . k[slot 1]
  }

  const int ncols = min(BLOCK_KV, p.T - k0);
  uint32_t kw[4] = {0u, 0u, 0u, 0u};
  if (live) {
    const uint4 kw4 = __ldg(reinterpret_cast<const uint4*>(p.keybits + (size_t)b * p.words + kb * 4));
    kw[0] = kw4.x; kw[1] = kw4.y; kw[2] = kw4.z; kw[3] = kw4.w;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int t = q0 + (int)(warp * 16 + g + 8 * r);
    if (t >= p.T) continue;
    float mneg = 0.f, inv = 0.f;
    if (live) {
      const size_t si = ((size_t)b * p.H + h) * p.T + t;
      mneg = -p.row_max[si] * LOG2E;
      const float l = p.row_sum[si];
      inv = l > 0.f ? 1.0f / l : 0.f;
      // esm2.py:135-139: rows of padded QUERY tokens are zero in the stacked result (padded key columns already are)
      if (p.zero_pad_rows && !((p.keybits[(size_t)b * p.words + (t >> 5)] >> (t & 31)) & 1u)) inv = 0.f;
    }
    float* dst = p.probs + (size_t)b * p.batch_stride + (size_t)h * p.T * p.T + (size_t)t * p.T + k0;
#pragma unroll
    for (int nb = 0; nb < 16; ++nb) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = nb * 8 + 2 * (int)c + e;
        if (key < ncols) dst[key] = masked_prob(s[nb][2 * r + e], kw[nb / 4], key, mneg, inv);
      }
    }
  }
}

template <int MODE>
inline cudaError_t launch_attention_probs_mode(const CUtensorMap& tmap_qkv, const ProbsParams& p, int n,
                                               cudaStream_t stream) {
  using namespace probs_cfg;
  constexpr int smem = smem_bytes(MODE ? 2 : 1);
  dim3 grid((p.T + BLOCK_KV - 1) / BLOCK_KV, (p.T + BLOCK_Q - 1) / BLOCK_Q, n * p.H);
  cudaError_t e = cudaFuncSetAttribute(attention_probs_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  return launch_pdl(attention_probs_kernel<MODE>, grid, dim3(NUM_THREADS), smem, stream, tmap_qkv, p);
}

// one launch over the n sequences p.b0 ... p.b0 + n - 1, n <= probs_cfg::seqs_per_launch(p.H): the caller splits a
// larger batch into launches of at most that many sequences
inline cudaError_t launch_attention_probs(const CUtensorMap& tmap_qkv, const ProbsParams& p, int n,
                                          cudaStream_t stream) {
  if (n <= 0 || n > probs_cfg::seqs_per_launch(p.H) || p.b0 < 0 || p.b0 + n > p.B) return cudaErrorInvalidValue;
  if (p.slots == 2) return launch_attention_probs_mode<2>(tmap_qkv, p, n, stream);
  if (p.lo_off > 0) return launch_attention_probs_mode<1>(tmap_qkv, p, n, stream);
  return launch_attention_probs_mode<0>(tmap_qkv, p, n, stream);
}

}  // namespace esmb200
