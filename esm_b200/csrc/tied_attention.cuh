// esm_b200 — MSA tied row attention (sm_90a, head_dim 64).
//
// Replaces esm/axial_attention.py:71-111 (RowSelfAttention.compute_attention_weights /
// compute_attention_update): the attention logits are SUMMED over the R alignment rows,
//     S[h,b,i,j] = sum_r sum_e q[b,r,i,h,e] * k[b,r,j,h,e]                      (einsum "rinhd,rjnhd->hnij", :87)
//     P = softmax_j(S)  (padded key columns filled with -10000, :94-97)          (:105)
//     ctx[b,r,i,h,:] = sum_j P[h,b,i,j] * v[b,r,j,h,:]                           (einsum "hnij,rjnhd->rinhd", :108)
// Both contractions read q/k/v IN PLACE from the fused projection output qkv [B*R*C, 3E] (fp16) through 2-D TMA boxes:
// for the logits the K loop simply walks over the rows r (row offset r*C, 64 K-elements per step), for the update the
// V tile of row r is the MN-major B operand, exactly like V in the flash-attention kernels.  No regrouping copies.
//
//   tied_scores_kernel : one CTA per (b, h, 128 query columns, 128 key columns); K = R*64; fp32 logits -> S [H,B,C,C]
//   tied_softmax_kernel: one warp per logits row; fp32 softmax; writes fp16 P [H*B*C, Cp] (Cp = C rounded up to 64,
//                        zero filled) and, on request, the fp32 probabilities in place of the logits
//   tied_pv_kernel     : one CTA per (b, h, 128 query columns, 4 alignment rows): D[128, 4 x 64] += P_tile V_r tile
//                        over the key columns; fp16 context -> ctx [B*R*C, E]
// Inside the MMA kernels (256 threads) thread 0 streams the operand tiles through a TMA ring (mbarrier completion) and
// all eight warps multiply with mma.sync from ldmatrix reads of the 128B-swizzled tiles.
//
// SPLIT ("fp32x3" precision): qkv is [B*R*C, 6E] = [q k v]_hi | [q k v]_lo, P is [H*B*C, 2*Cp] (hi | lo rows) and ctx is
// [B*R*C, 2E] (hi | lo); every product runs hi*hi + lo*hi + hi*lo into fp32.  Every stage then carries both halves of
// its tiles, so the logits ring drops to 3 stages.  The logits contraction is K = R*64 long (65,536 at R = 1024): each
// alignment row's 64-wide slab is accumulated in a fresh fragment and added to the running sum with ordinary fp32 adds,
// so the tensor core's truncating accumulation only ever sums 3 x 64 products (DESIGN.md section 4).
#pragma once

#include "attention_common.cuh"

namespace esmb200 {

struct TiedParams {
  int B, R, C, H, E;   // E = 64 * H
  int Cp;              // C rounded up to 64: row pitch of P
  float* S;            // [H, B, C, C] fp32 logits (tied_scores) / probabilities (tied_softmax, optional)
  __half* P;           // [H*B*C, Cp] fp16 probabilities (SPLIT: [H*B*C, 2*Cp], hi | lo)
  __half* ctx;         // [B*R*C, E] (SPLIT: [B*R*C, 2E], hi | lo)
  const uint8_t* key_pad;  // optional: key_pad[b * key_pad_stride + c] = 1 <=> key column c of alignment b is padding
                           // (filled with -10000 before the softmax)
  long long key_pad_stride;
  int write_probs;     // tied_softmax: also write the fp32 probabilities over S
};

namespace tied_cfg {
constexpr int NUM_THREADS = 256;
// scores: 8 warps as 4 (rows) x 2 (columns), warp tile 32 x 64
constexpr int S_BM = 128, S_BN = 128, S_STAGES = 4;
constexpr int S_A_BYTES = S_BM * 128, S_B_BYTES = S_BN * 128;
constexpr int S_STAGE_BYTES = S_A_BYTES + S_B_BYTES;                 // 32 KB
constexpr int S_SMEM_BYTES = S_STAGES * S_STAGE_BYTES + 1024 + 256;
constexpr int S_STAGES_SPLIT = 3;                                    // 64 KB stages: Q and K, hi and lo
constexpr int S_SMEM_BYTES_SPLIT = S_STAGES_SPLIT * 2 * S_STAGE_BYTES + 1024 + 256;
// update: warp w owns query rows [16 w, 16 w + 16) of every alignment row of the CTA
constexpr int V_BM = 128, V_ROWS = 4, V_STAGES = 2;
constexpr int V_P_BYTES = V_BM * 128, V_V_BYTES = 64 * 128;          // 16 KB + 4 x 8 KB
constexpr int V_STAGE_BYTES = V_P_BYTES + V_ROWS * V_V_BYTES;        // 48 KB
constexpr int V_SMEM_BYTES = V_STAGES * V_STAGE_BYTES + 1024 + 256;
constexpr int V_SMEM_BYTES_SPLIT = V_STAGES * 2 * V_STAGE_BYTES + 1024 + 256;  // 96 KB stages: P and V, hi and lo
}  // namespace tied_cfg

// ---------------------------------------------------------------------------------------------------------------
// S = sum_r Q_r K_r^T
// ---------------------------------------------------------------------------------------------------------------
template <bool SPLIT>
__global__ void __launch_bounds__(tied_cfg::NUM_THREADS, 1)
tied_scores_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                   const TiedParams p) {
  using namespace tied_cfg;
  // stage s: [Q_hi | K_hi] (+ [Q_lo | K_lo] S_STAGE_BYTES further on with SPLIT)
  constexpr int STAGES = SPLIT ? S_STAGES_SPLIT : S_STAGES;
  constexpr int STAGE_BYTES = (SPLIT ? 2 : 1) * S_STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);  // [STAGES]

  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = lane / 4, c = lane % 4;
  const uint32_t wm = warp % 4, wn = warp / 4;
  const int m0 = blockIdx.x * S_BM, n0 = blockIdx.y * S_BN;
  const int b = blockIdx.z / p.H, h = blockIdx.z % p.H;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    for (int i = 0; i < STAGES; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  auto load = [&](int r) {
    const int s = r % STAGES;
    const int row = (b * p.R + r) * p.C;
    mbar_arrive_expect_tx(&full[s], STAGE_BYTES);
    tma_load_2d(smem + s * STAGE_BYTES, &tmap_q, &full[s], h * 64, row + m0);
    tma_load_2d(smem + s * STAGE_BYTES + S_A_BYTES, &tmap_k, &full[s], p.E + h * 64, row + n0);
    if constexpr (SPLIT) {  // the lo halves, 3E columns to the right
      tma_load_2d(smem + s * STAGE_BYTES + S_STAGE_BYTES, &tmap_q, &full[s], 3 * p.E + h * 64, row + m0);
      tma_load_2d(smem + s * STAGE_BYTES + S_STAGE_BYTES + S_A_BYTES, &tmap_k, &full[s], 4 * p.E + h * 64, row + n0);
    }
  };
  if (threadIdx.x == 0)
    for (int r = 0; r < STAGES && r < p.R; ++r) load(r);

  float acc[2][8][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[mi][i][0] = acc[mi][i][1] = acc[mi][i][2] = acc[mi][i][3] = 0.f;
  for (int r = 0; r < p.R; ++r) {
    const int s = r % STAGES;
    mbar_wait(&full[s], (r / STAGES) & 1);
    const uint32_t st = smem_u32(smem + s * STAGE_BYTES);
    if constexpr (SPLIT) {
      // row r's slab in a fresh fragment (lo terms first), then one fp32 add per element into the running sum
      const uint32_t lo = st + S_STAGE_BYTES;
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        float part[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i) part[i][0] = part[i][1] = part[i][2] = part[i][3] = 0.f;
        const uint32_t qr = wm * 32 + mi * 16;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          uint32_t ah[4], al[4];
          ldsm_a(st, qr, kk, ah);
          ldsm_a(lo, qr, kk, al);
#pragma unroll
          for (int n2 = 0; n2 < 4; ++n2) {
            uint32_t bh[4], bl[4];
            ldsm_b(st + S_A_BYTES, wn * 64 + 16 * n2, kk, bh);
            ldsm_b(lo + S_A_BYTES, wn * 64 + 16 * n2, kk, bl);
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {  // q_lo k_hi + q_hi k_lo + q_hi k_hi
              mma16816(part[2 * n2 + hf], al, bh[2 * hf], bh[2 * hf + 1]);
              mma16816(part[2 * n2 + hf], ah, bl[2 * hf], bl[2 * hf + 1]);
              mma16816(part[2 * n2 + hf], ah, bh[2 * hf], bh[2 * hf + 1]);
            }
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[mi][i][e] += part[i][e];
      }
    } else {
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) qk_tile<8>(acc[mi], st, wm * 32 + mi * 16, st + S_A_BYTES, wn * 64);
    }
    __syncthreads();  // every warp is done with stage s
    if (threadIdx.x == 0 && r + STAGES < p.R) load(r + STAGES);
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int ci = m0 + (int)(wm * 32 + mi * 16 + g + 8 * hr);
      if (ci >= p.C) continue;
      float* dst = p.S + ((size_t)(h * p.B + b) * p.C + ci) * p.C;
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int cj = n0 + (int)(wn * 64 + nb * 8 + 2 * c) + e;
          if (cj < p.C) dst[cj] = acc[mi][nb][2 * hr + e];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// row softmax over the key columns: fp32 in, fp16 P out (+ fp32 probabilities in place when asked); SPLIT: P rows
// are hi | lo, [H*B*C, 2*Cp]
// ---------------------------------------------------------------------------------------------------------------
constexpr int TIED_MAX_C = 1024;  // MSA Transformer max_positions (msa_transformer.py:57-60)

// (SPLIT: at ptxas's default register target of 64 the hi | lo store spills 4 bytes; one block per SM lifts it to 71)
template <bool SPLIT>
__global__ void __launch_bounds__(256, SPLIT ? 1 : 0)
tied_softmax_kernel(const TiedParams p) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const long long row = (long long)blockIdx.x * 8 + warp;  // (h*B + b)*C + ci
  const long long rows = (long long)p.H * p.B * p.C;
  if (row >= rows) return;
  pdl_launch_dependents();
  pdl_wait();
  const int b = (int)((row / p.C) % p.B);
  float* s = p.S + row * p.C;
  const uint8_t* pad = p.key_pad ? p.key_pad + (size_t)b * p.key_pad_stride : nullptr;
  float v[TIED_MAX_C / 32];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < TIED_MAX_C / 32; ++i) {
    const int c = i * 32 + lane;
    float x = -INFINITY;
    if (c < p.C) {
      x = s[c];
      if (pad && pad[c]) x = -10000.f;  // axial_attention.py:94-97
    }
    v[i] = x;
    mx = fmaxf(mx, x);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < TIED_MAX_C / 32; ++i) {
    v[i] = (i * 32 + lane < p.C) ? __expf(v[i] - mx) : 0.f;
    sum += v[i];
  }
  sum = warp_sum(sum);
  const float inv = 1.0f / sum;
  __half* pr = p.P + row * (SPLIT ? 2 * p.Cp : p.Cp);
#pragma unroll
  for (int i = 0; i < TIED_MAX_C / 32; ++i) {
    const int c = i * 32 + lane;
    if (c < p.Cp) {
      const float q = v[i] * inv;
      const __half qh = __float2half_rn(q);
      pr[c] = qh;
      if constexpr (SPLIT) pr[p.Cp + c] = __float2half_rn(q - __half2float(qh));
      if (p.write_probs && c < p.C) s[c] = q;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// ctx_r = P V_r for 4 alignment rows r per CTA
// ---------------------------------------------------------------------------------------------------------------
template <bool SPLIT>
__global__ void __launch_bounds__(tied_cfg::NUM_THREADS, 1)
tied_pv_kernel(const __grid_constant__ CUtensorMap tmap_p, const __grid_constant__ CUtensorMap tmap_v,
               const TiedParams p) {
  using namespace tied_cfg;
  // stage s: [P_hi | V_hi x 4] (+ [P_lo | V_lo x 4] V_STAGE_BYTES further on with SPLIT)
  constexpr int STAGE_BYTES = (SPLIT ? 2 : 1) * V_STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + V_STAGES * STAGE_BYTES);  // [V_STAGES]

  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = lane / 4, c = lane % 4;
  const int m0 = blockIdx.x * V_BM;
  const int r0 = blockIdx.y * V_ROWS;
  const int nr = min(V_ROWS, p.R - r0);
  const int b = blockIdx.z / p.H, h = blockIdx.z % p.H;
  const int nk = p.Cp / 64;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_p);
    tma_prefetch_desc(&tmap_v);
    for (int i = 0; i < V_STAGES; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  auto load = [&](int j) {
    const int s = j % V_STAGES;
    uint8_t* st = smem + s * STAGE_BYTES;
    mbar_arrive_expect_tx(&full[s], (SPLIT ? 2 : 1) * (V_P_BYTES + nr * V_V_BYTES));
    tma_load_2d(st, &tmap_p, &full[s], j * 64, (h * p.B + b) * p.C + m0);
    for (int i = 0; i < nr; ++i)
      tma_load_2d(st + V_P_BYTES + i * V_V_BYTES, &tmap_v, &full[s], 2 * p.E + h * 64, (b * p.R + r0 + i) * p.C + j * 64);
    if constexpr (SPLIT) {  // P_lo Cp columns, v_lo 3E columns to the right
      tma_load_2d(st + V_STAGE_BYTES, &tmap_p, &full[s], p.Cp + j * 64, (h * p.B + b) * p.C + m0);
      for (int i = 0; i < nr; ++i)
        tma_load_2d(st + V_STAGE_BYTES + V_P_BYTES + i * V_V_BYTES, &tmap_v, &full[s], 5 * p.E + h * 64,
                    (b * p.R + r0 + i) * p.C + j * 64);
    }
  };
  if (threadIdx.x == 0)
    for (int j = 0; j < V_STAGES && j < nk; ++j) load(j);

  float acc[V_ROWS][8][4];
#pragma unroll
  for (int i = 0; i < V_ROWS; ++i)
#pragma unroll
    for (int n = 0; n < 8; ++n) acc[i][n][0] = acc[i][n][1] = acc[i][n][2] = acc[i][n][3] = 0.f;
  for (int j = 0; j < nk; ++j) {
    const int s = j % V_STAGES;
    mbar_wait(&full[s], (j / V_STAGES) & 1);
    const uint32_t st = smem_u32(smem + s * STAGE_BYTES);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      ldsm_a(st, warp * 16, kk, a);
      [[maybe_unused]] uint32_t al[4];  // SPLIT: P_lo
      if constexpr (SPLIT) ldsm_a(st + V_STAGE_BYTES, warp * 16, kk, al);
#pragma unroll
      for (int i = 0; i < V_ROWS; ++i) {
        if (i >= nr) break;
#pragma unroll
        for (int n2 = 0; n2 < 4; ++n2) {
          uint32_t bv[4];
          ldsm_bt(st + V_P_BYTES + i * V_V_BYTES, kk, 16 * n2, bv);
          mma16816(acc[i][2 * n2], a, bv[0], bv[1]);
          mma16816(acc[i][2 * n2 + 1], a, bv[2], bv[3]);
          if constexpr (SPLIT) {  // + p_lo v_hi + p_hi v_lo
            mma16816(acc[i][2 * n2], al, bv[0], bv[1]);
            mma16816(acc[i][2 * n2 + 1], al, bv[2], bv[3]);
            uint32_t bl[4];
            ldsm_bt(st + V_STAGE_BYTES + V_P_BYTES + i * V_V_BYTES, kk, 16 * n2, bl);
            mma16816(acc[i][2 * n2], a, bl[0], bl[1]);
            mma16816(acc[i][2 * n2 + 1], a, bl[2], bl[3]);
          }
        }
      }
    }
    __syncthreads();  // every warp is done with stage s
    if (threadIdx.x == 0 && j + V_STAGES < nk) load(j + V_STAGES);
  }
#pragma unroll
  for (int i = 0; i < V_ROWS; ++i) {
    if (i >= nr) break;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int ci = m0 + (int)(warp * 16 + g + 8 * hr);
      if (ci >= p.C) continue;
      __half* dst = p.ctx + ((size_t)(b * p.R + r0 + i) * p.C + ci) * (SPLIT ? 2 * p.E : p.E) + h * 64;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const __half2 h2 = __floats2half2_rn(acc[i][n][2 * hr], acc[i][n][2 * hr + 1]);
        *reinterpret_cast<__half2*>(dst + n * 8 + 2 * c) = h2;
        if constexpr (SPLIT) {  // ctx [M, 2E]: lo half E columns to the right
          const float2 f = __half22float2(h2);
          *reinterpret_cast<__half2*>(dst + p.E + n * 8 + 2 * c) =
              __floats2half2_rn(acc[i][n][2 * hr] - f.x, acc[i][n][2 * hr + 1] - f.y);
        }
      }
    }
  }
}

template <bool SPLIT>
inline cudaError_t launch_tied_scores(const CUtensorMap& tq, const CUtensorMap& tk, const TiedParams& p,
                                      cudaStream_t st) {
  using namespace tied_cfg;
  constexpr int smem = SPLIT ? S_SMEM_BYTES_SPLIT : S_SMEM_BYTES;
  cudaError_t e = cudaFuncSetAttribute(tied_scores_kernel<SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  dim3 grid((p.C + S_BM - 1) / S_BM, (p.C + S_BN - 1) / S_BN, p.B * p.H);
  return launch_pdl(tied_scores_kernel<SPLIT>, grid, dim3(NUM_THREADS), smem, st, tq, tk, p);
}

template <bool SPLIT>
inline cudaError_t launch_tied_softmax(const TiedParams& p, cudaStream_t st) {
  const long long rows = (long long)p.H * p.B * p.C;
  return launch_pdl(tied_softmax_kernel<SPLIT>, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, st, p);
}

template <bool SPLIT>
inline cudaError_t launch_tied_pv(const CUtensorMap& tp, const CUtensorMap& tv, const TiedParams& p, cudaStream_t st) {
  using namespace tied_cfg;
  constexpr int smem = SPLIT ? V_SMEM_BYTES_SPLIT : V_SMEM_BYTES;
  cudaError_t e = cudaFuncSetAttribute(tied_pv_kernel<SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  dim3 grid((p.C + V_BM - 1) / V_BM, (p.R + V_ROWS - 1) / V_ROWS, p.B * p.H);
  return launch_pdl(tied_pv_kernel<SPLIT>, grid, dim3(NUM_THREADS), smem, st, tp, tv, p);
}

}  // namespace esmb200
