// esm_b200 — need_head_weights + return_contacts in ONE pass (sm_90a, head_dim <= 64, or <= 128 with DS = 2): the
// attention probabilities of a layer are written to the stacked [B,L,H,T,T] result AND folded into the contact head's
// accumulators while they are still in registers, so the 4*B*L*H*T^2-byte stack is written once and never read back.
// The STORE = false instantiation (esmb200_stack_contacts: contacts without the stack) is the same pass without the
// probability stores: same tiles, same masked_prob arithmetic, same accumulation order, so its acc, row_part and
// col_part are bit-identical to the storing pass's, and the caller never allocates the stack.
//
// Replaces esm/multihead_attention.py:397-400 (per-head probabilities) and the per-layer share of
// ContactPredictionHead.forward, esm/modules.py:338-357 (eos masking, bos/eos crop, symmetrize :27-29, apc :32-41), in
// the restated form of elementwise.cuh: with A_h the masked, cropped map of head h,
//     acc[b,i,j]        += sum_h w_h A_h[i,j]                  (one owner CTA per tile: plain read-modify-write)
//     row_part[b,h,4kt+c,i] = sum_{j in 32-key quarter c of key tile kt} A_h[i,j]   (partials, summed by the caller)
//     col_part[b,h,4qt+r,j] = sum_{i in 32-row quarter r of query tile qt} A_h[i,j]   (partials, summed by the caller)
// No atomics: every output element has one writer and every sum a fixed order -> bit-reproducible contacts.
//
// One CTA = (128-key tile, 128-query tile, sequence) and LOOPS OVER THE HEADS: thread 0 streams the (Q_h, K_h) tiles
// through a 2-stage TMA ring; eight warps (16 query rows x 128 keys each) compute S_h = Q_h K_h^T with mma.sync, turn
// it into p = exp(s - m) / l with the statistics saved by the forward kernel and accumulate in registers.
#pragma once

#include "attention_common.cuh"

namespace esmb200 {

struct ContactFuseParams {
  int B, T, H, E;            // E = 64 * slots * H
  int slots = 1;             // 64-wide column slots per head (2: head_dim <= 128, S_h sums both slots)
  const uint32_t* keybits;   // [B, words]
  const int* kvlen;          // [B]
  int words;
  const float* row_max;      // [B,H,T] reference max / row sum of the forward kernel
  const float* row_sum;
  float* probs;              // this layer's slice of the stacked result: batch b at probs + b * batch_stride; NULL:
                             // contacts only (the STORE = false instantiation)
  long long batch_stride;
  int zero_pad_rows;
  // contact head
  const float* w;            // [H] regression weights of this layer's heads
  const uint8_t* keep;       // [B,T] 1 = not <eos>, or NULL
  float* acc;                // [B,S,S]
  float* row_part;           // [B,H,4*nkt,S]
  float* col_part;           // [B,H,4*nqt,S]
  int lo, S;                 // cropped positions [lo, lo+S)
};

namespace cfuse_cfg {
constexpr int BLOCK = 128;            // query rows and keys per tile
constexpr int NUM_THREADS = 256;      // eight warps of 16 query rows x 128 keys
constexpr int STAGES = 2;
constexpr int TILE_BYTES = attn_cfg::TILE_BYTES;
constexpr int smem_bytes(int ds) {  // ds operand tiles per Q and per K stage
  return STAGES * 2 * ds * TILE_BYTES + 1024 /*align*/ + 64 /*barriers*/ + 2 * 8 * BLOCK * 4 /*column sums*/;
}
}  // namespace cfuse_cfg

template <int DS, bool STORE>  // STORE = false: p.probs and p.batch_stride are not read, no probability is written
__global__ void __launch_bounds__(cfuse_cfg::NUM_THREADS, 1)
attention_probs_contact_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const ContactFuseParams p) {
  using namespace cfuse_cfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int STAGE_BYTES = DS * TILE_BYTES;        // Q (or K) tiles of one head: one per 64-wide slot
  uint8_t* smem_q = smem;                             // [STAGES][DS]
  uint8_t* smem_k = smem + STAGES * STAGE_BYTES;      // [STAGES][DS]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * 2 * STAGE_BYTES);  // [STAGES] TMA -> warps
  float* colsum = reinterpret_cast<float*>(smem + STAGES * 2 * STAGE_BYTES + 64);  // [2 (head parity)][8 warps][128]

  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = lane / 4, c = lane % 4;
  const int kt = blockIdx.x, qt = blockIdx.y, b = blockIdx.z;
  const int q0 = qt * BLOCK, k0 = kt * BLOCK;
  const int row_base = b * p.T;
  const int nkt = gridDim.x, nqt = gridDim.y;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  const bool live = k0 < p.kvlen[b];  // otherwise every key of this tile is masked: all probabilities are exactly 0
  auto load = [&](int h) {
    const int s = h % STAGES;
    mbar_arrive_expect_tx(&full[s], 2 * STAGE_BYTES);
#pragma unroll
    for (int sl = 0; sl < DS; ++sl) {
      tma_load_2d(smem_q + s * STAGE_BYTES + sl * TILE_BYTES, &tmap_qkv, &full[s], (h * DS + sl) * 64, row_base + q0);
      tma_load_2d(smem_k + s * STAGE_BYTES + sl * TILE_BYTES, &tmap_qkv, &full[s], p.E + (h * DS + sl) * 64,
                  row_base + k0);
    }
  };
  if (live && threadIdx.x == 0)
    for (int h = 0; h < STAGES && h < p.H; ++h) load(h);

  const int hi = p.lo + p.S;
  const uint8_t* kp = p.keep ? p.keep + (size_t)b * p.T : nullptr;
  const int ncols = min(BLOCK, p.T - k0);
  // rows of this thread: t[r] = q0 + 16 warp + g + 8 r; contact masks: position kept (not <eos>) and inside the crop
  int t[2];
  bool row_ok[2], ri[2], qpad[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    t[r] = q0 + (int)(warp * 16 + g + 8 * r);
    row_ok[r] = t[r] < p.T;
    ri[r] = row_ok[r] && t[r] >= p.lo && t[r] < hi && (!kp || kp[t[r]]);
    qpad[r] = p.zero_pad_rows && row_ok[r] && !((p.keybits[(size_t)b * p.words + (t[r] >> 5)] >> (t[r] & 31)) & 1u);
  }
  // columns of this thread: key k0 + 8 nb + 2 c + e
  uint32_t cmask = 0u;  // bit 2 nb + e: column kept and inside the crop
#pragma unroll
  for (int nb = 0; nb < 16; ++nb)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int j = k0 + nb * 8 + 2 * (int)c + e;
      if (j < p.T && j >= p.lo && j < hi && (!kp || kp[j])) cmask |= 1u << (2 * nb + e);
    }
  uint32_t kw[4] = {0u, 0u, 0u, 0u};
  if (live) {
    const uint4 kw4 = __ldg(reinterpret_cast<const uint4*>(p.keybits + (size_t)b * p.words + kt * 4));
    kw[0] = kw4.x; kw[1] = kw4.y; kw[2] = kw4.z; kw[3] = kw4.w;
  }
  float acc[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;

  for (int h = 0; h < p.H; ++h) {
    const int s = h % STAGES;
    const float wh = __ldg(p.w + h);
    float sc[16][4];
#pragma unroll
    for (int i = 0; i < 16; ++i) sc[i][0] = sc[i][1] = sc[i][2] = sc[i][3] = 0.f;
    if (live) {
      mbar_wait(&full[s], (h / STAGES) & 1);
#pragma unroll
      for (int sl = 0; sl < DS; ++sl)
        qk_tile<16>(sc, smem_u32(smem_q + s * STAGE_BYTES + sl * TILE_BYTES), warp * 16,
                    smem_u32(smem_k + s * STAGE_BYTES + sl * TILE_BYTES), 0);
    }
    float rs[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};  // row partials per 32-key quarter
    float cs[16][2];                                               // column sums of this warp's 16 rows
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mneg = 0.f, inv = 0.f;
      if (live && row_ok[r]) {
        const size_t si = ((size_t)b * p.H + h) * p.T + t[r];
        mneg = -p.row_max[si] * attn_cfg::LOG2E;
        const float l = p.row_sum[si];
        inv = (l > 0.f && !qpad[r]) ? 1.0f / l : 0.f;  // esm2.py:135-139: rows of padded query tokens are zero
      }
      float* dst = STORE ? p.probs + (size_t)b * p.batch_stride + (size_t)h * p.T * p.T + (size_t)t[r] * p.T + k0
                         : nullptr;
#pragma unroll
      for (int nb = 0; nb < 16; ++nb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = nb * 8 + 2 * (int)c + e;
          const float pr = live ? masked_prob(sc[nb][2 * r + e], kw[nb / 4], key, mneg, inv) : 0.f;
          if (STORE && row_ok[r] && key < ncols) dst[key] = pr;
          const float x = (ri[r] && ((cmask >> (2 * nb + e)) & 1u)) ? pr : 0.f;
          acc[nb][2 * r + e] = fmaf(wh, x, acc[nb][2 * r + e]);
          rs[r][nb / 4] += x;
          if (r == 0) cs[nb][e] = x;
          else cs[nb][e] += x;
        }
    }
    // row partial of each 32-key quarter (4 * nkt partials per row)
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float v = quad_sum(rs[r][q]);
        if (c == 0 && row_ok[r] && t[r] >= p.lo && t[r] < hi)
          p.row_part[(((size_t)b * p.H + h) * (4 * nkt) + 4 * kt + q) * p.S + (t[r] - p.lo)] = v;  // 0 for <eos>
      }
    // column sums over the warp's 16 rows (lanes of equal c), then over the two warps of a 32-row quarter
    float* cw = colsum + ((h & 1) * 8 + warp) * BLOCK;
#pragma unroll
    for (int nb = 0; nb < 16; ++nb)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float v = cs[nb][e];
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 8);
        v += __shfl_xor_sync(0xffffffffu, v, 16);
        if (g == 0) cw[nb * 8 + 2 * c + e] = v;
      }
    __syncthreads();  // every warp is done with stage s and has written its column sums
    if (live && threadIdx.x == 0 && h + STAGES < p.H) load(h + STAGES);
    const float* cr = colsum + (h & 1) * 8 * BLOCK;
    for (int i = threadIdx.x; i < 4 * BLOCK; i += NUM_THREADS) {
      const int rq = i / BLOCK, col = i % BLOCK, j = k0 + col;
      if (j >= p.lo && j < hi && j < p.T)  // (4 * nqt partials per column; 0 for <eos> columns)
        p.col_part[(((size_t)b * p.H + h) * (4 * nqt) + 4 * qt + rq) * p.S + (j - p.lo)] =
            cr[(2 * rq) * BLOCK + col] + cr[(2 * rq + 1) * BLOCK + col];
    }
  }
  // acc tile: this CTA is the only writer of acc[b, rows of qt, columns of kt]; layers are separate launches
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!ri[r]) continue;
    float* dst = p.acc + ((size_t)b * p.S + (t[r] - p.lo)) * p.S;
#pragma unroll
    for (int nb = 0; nb < 16; ++nb)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = k0 + nb * 8 + 2 * (int)c + e;
        if (j >= p.lo && j < hi && j < p.T) dst[j - p.lo] += acc[nb][2 * r + e];
      }
  }
}

template <int DS, bool STORE>
inline cudaError_t launch_attention_probs_contact_ds(const CUtensorMap& tmap_qkv, const ContactFuseParams& p,
                                                     cudaStream_t stream) {
  using namespace cfuse_cfg;
  constexpr int smem = smem_bytes(DS);
  cudaError_t e = cudaFuncSetAttribute(attention_probs_contact_kernel<DS, STORE>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  dim3 grid((p.T + BLOCK - 1) / BLOCK, (p.T + BLOCK - 1) / BLOCK, p.B);
  return launch_pdl(attention_probs_contact_kernel<DS, STORE>, grid, dim3(NUM_THREADS), smem, stream, tmap_qkv, p);
}

// p.probs == NULL: the store-free pass (contacts only)
inline cudaError_t launch_attention_probs_contact(const CUtensorMap& tmap_qkv, const ContactFuseParams& p,
                                                  cudaStream_t stream) {
  if (p.probs)
    return p.slots == 2 ? launch_attention_probs_contact_ds<2, true>(tmap_qkv, p, stream)
                        : launch_attention_probs_contact_ds<1, true>(tmap_qkv, p, stream);
  return p.slots == 2 ? launch_attention_probs_contact_ds<2, false>(tmap_qkv, p, stream)
                      : launch_attention_probs_contact_ds<1, false>(tmap_qkv, p, stream);
}

}  // namespace esmb200
