// esm_b200 — attention forward (sm_90a): flash attention with TMA-fed K/V stages and warp-level tensor-core MMAs, for
// the inputs the warpgroup kernel (attention_wg.cuh) does not take: fp32x3 operands and 128-wide heads.
//
// Replaces esm/multihead_attention.py:357-394.  One CTA per (sequence, head, 128-query tile), eight warps of 16 query
// rows each.  Thread 0 loads the Q tile once and streams 64-key K/V blocks through a two-stage TMA ring (mbarrier
// completion); every warp computes S = Q K^T for its rows (mma.sync m16n8k16 from ldmatrix reads of the 128B-swizzled
// tiles), applies the key-padding mask, keeps the online-softmax statistics in registers (exact running maximum, fp32
// row sums), rescales O, and multiplies P (fp16, straight from the S registers) with V (ldmatrix.trans).
// Exactness: P is rounded to fp16 relative to the running maximum (values <= 1), row sums and O are fp32.
//
// DS = 2 (64 < head_dim <= 128, ESM-2 15B): a head is TWO 64-wide slots (elementwise.cuh head_slot); S sums both slots,
// O has a half per slot.  SPLIT ("fp32x3" precision): q, k, v and P are fp16 hi | lo pairs and every product runs
// hi*hi + lo*hi + hi*lo into the same fp32 accumulator.
#pragma once

#include "attention_common.cuh"
#include "attention_wg.cuh"

namespace esmb200 {

namespace attn8_cfg {
constexpr int BLOCK_Q = 128;
constexpr int BLOCK_KV = 64;
constexpr int HEAD_DIM = 64;
constexpr int KV_STAGES = 2;
constexpr int Q_BYTES = 128 * 64 * 2;  // 16 KB
constexpr int KV_BYTES = 64 * 64 * 2;  // 8 KB per K tile and per V tile
constexpr int NUM_THREADS = 256;
constexpr int smem_bytes(int np) { return np * Q_BYTES + KV_STAGES * 2 * np * KV_BYTES + 1024 + 64; }
}  // namespace attn8_cfg

template <bool SPLIT, int DS>
__global__ void __launch_bounds__(attn8_cfg::NUM_THREADS, (SPLIT || DS == 2) ? 1 : 2)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv,
                     const AttnParams p) {
  using namespace attn8_cfg;
  constexpr float LOG2E = attn_cfg::LOG2E;
  static_assert(!(SPLIT && DS == 2), "fp32x3 operands and two-slot heads are not combined");
  constexpr int NP = (SPLIT || DS == 2) ? 2 : 1;  // operand tiles per Q / K / V: hi (+ lo), or slot 0 (+ slot 1)
  constexpr int HEAD_COLS = HEAD_DIM * DS;        // columns of one head in qkv / ctx
  constexpr int KB = NP * KV_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;                                 // [NP]
  uint8_t* smem_k = smem + NP * Q_BYTES;                  // [KV_STAGES][NP]
  uint8_t* smem_v = smem + NP * Q_BYTES + KV_STAGES * KB;  // [KV_STAGES][NP]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NP * Q_BYTES + 2 * KV_STAGES * KB);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;  // [KV_STAGES]

  const int nqt = (p.T + BLOCK_Q - 1) / BLOCK_Q;
  const int w = blockIdx.x;
  const int qt = w % nqt, h = (w / nqt) % p.H, b = w / (nqt * p.H);
  const int row_base = (b / p.cols) * p.T;
  const int x0 = (b % p.cols) * (SPLIT ? 6 : 3) * p.E + h * HEAD_COLS;  // SPLIT: a token's qkv is 6E wide (hi | lo)
  const int part_off = SPLIT ? p.lo_off : HEAD_DIM;  // column distance of the second operand tile
  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = lane / 4, c = lane % 4;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_kv);
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_STAGES; ++i) mbar_init(&kv_full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // everything below reads the previous kernel's output (qkv, key bits) or writes ctx
  const int nblk = (p.kvlen[b] + BLOCK_KV - 1) / BLOCK_KV;

  auto load_kv = [&](int j) {
    const int s = j % KV_STAGES;
    mbar_arrive_expect_tx(&kv_full[s], 2 * KB);
#pragma unroll
    for (int part = 0; part < NP; ++part) {
      tma_load_2d(smem_k + s * KB + part * KV_BYTES, &tmap_kv, &kv_full[s], x0 + p.E + part * part_off,
                  row_base + j * BLOCK_KV);
      tma_load_2d(smem_v + s * KB + part * KV_BYTES, &tmap_kv, &kv_full[s], x0 + 2 * p.E + part * part_off,
                  row_base + j * BLOCK_KV);
    }
  };
  if (threadIdx.x == 0 && nblk > 0) {
    mbar_arrive_expect_tx(q_full, NP * Q_BYTES);
#pragma unroll
    for (int part = 0; part < NP; ++part)
      tma_load_2d(smem_q + part * Q_BYTES, &tmap_q, q_full, x0 + part * part_off, row_base + qt * BLOCK_Q);
    for (int j = 0; j < KV_STAGES && j < nblk; ++j) load_kv(j);
  }

  const uint32_t q_base = smem_u32(smem_q), k_base = smem_u32(smem_k), v_base = smem_u32(smem_v);
  const uint32_t qrow = warp * 16;
  const uint32_t* kb_ptr = p.keybits + (size_t)b * p.words;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[DS][8][4];
#pragma unroll
  for (int sl = 0; sl < DS; ++sl)
#pragma unroll
    for (int i = 0; i < 8; ++i) o[sl][i][0] = o[sl][i][1] = o[sl][i][2] = o[sl][i][3] = 0.f;

  if (nblk > 0) mbar_wait(q_full, 0);
  for (int j = 0; j < nblk; ++j) {
    const int s = j % KV_STAGES;
    const uint2 kw2 = __ldg(reinterpret_cast<const uint2*>(kb_ptr + j * 2));
    mbar_wait(&kv_full[s], (j / KV_STAGES) & 1);
    const uint32_t kst = k_base + s * KB, vst = v_base + s * KB;
    float sc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) sc[i][0] = sc[i][1] = sc[i][2] = sc[i][3] = 0.f;
    qk_tile<8>(sc, q_base, qrow, kst, 0);
    if constexpr (SPLIT) {  // + q_lo k_hi + q_hi k_lo
      qk_tile<8>(sc, q_base + Q_BYTES, qrow, kst, 0);
      qk_tile<8>(sc, q_base, qrow, kst + KV_BYTES, 0);
    }
    if constexpr (DS == 2) qk_tile<8>(sc, q_base + Q_BYTES, qrow, kst + KV_BYTES, 0);  // + q[slot 1] . k[slot 1]

    // key-padding mask, running maximum, rescale
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      const uint32_t wd = nb < 4 ? kw2.x : kw2.y;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const uint32_t key = (nb % 4) * 8 + 2 * c + e;
        if (!((wd >> key) & 1u)) sc[nb][e] = sc[nb][2 + e] = -INFINITY;
        mx[0] = fmaxf(mx[0], sc[nb][e]);
        mx[1] = fmaxf(mx[1], sc[nb][2 + e]);
      }
    }
    float ref[2], alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float mn = fmaxf(m[r], quad_max(mx[r]));
      alpha[r] = (mn == -INFINITY) ? 1.f : ex2_approx((m[r] - mn) * LOG2E);  // ex2(-inf) = 0 before the first key
      m[r] = mn;
      ref[r] = (mn == -INFINITY) ? 0.f : -mn * LOG2E;
      l[r] *= alpha[r];
    }
#pragma unroll
    for (int sl = 0; sl < DS; ++sl)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        o[sl][i][0] *= alpha[0]; o[sl][i][1] *= alpha[0];
        o[sl][i][2] *= alpha[1]; o[sl][i][3] *= alpha[1];
      }
    uint32_t ph[8][2];
    [[maybe_unused]] uint32_t pl[8][2];  // SPLIT: lo halves of P
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float p0 = ex2_approx(fmaf(sc[nb][2 * r], LOG2E, ref[r]));
        const float p1 = ex2_approx(fmaf(sc[nb][2 * r + 1], LOG2E, ref[r]));
        l[r] += p0 + p1;
        const __half2 h2 = __floats2half2_rn(p0, p1);
        ph[nb][r] = *reinterpret_cast<const uint32_t*>(&h2);
        if constexpr (SPLIT) {
          const float2 f = __half22float2(h2);
          pl[nb][r] = pack_half2(p0 - f.x, p1 - f.y);
        }
      }
    }
    // O += P V: A fragment of keys [16 kk, 16 kk + 16) = S blocks 2 kk, 2 kk + 1
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t a[4] = {ph[2 * kk][0], ph[2 * kk][1], ph[2 * kk + 1][0], ph[2 * kk + 1][1]};
      [[maybe_unused]] uint32_t al[4];
      if constexpr (SPLIT) {
        al[0] = pl[2 * kk][0]; al[1] = pl[2 * kk][1]; al[2] = pl[2 * kk + 1][0]; al[3] = pl[2 * kk + 1][1];
      }
#pragma unroll
      for (int n2 = 0; n2 < 4; ++n2) {
        uint32_t bv[4];
        ldsm_bt(vst, kk, 16 * n2, bv);
        mma16816(o[0][2 * n2], a, bv[0], bv[1]);
        mma16816(o[0][2 * n2 + 1], a, bv[2], bv[3]);
        if constexpr (SPLIT) {  // + p_lo v_hi + p_hi v_lo
          mma16816(o[0][2 * n2], al, bv[0], bv[1]);
          mma16816(o[0][2 * n2 + 1], al, bv[2], bv[3]);
          uint32_t bl[4];
          ldsm_bt(vst + KV_BYTES, kk, 16 * n2, bl);
          mma16816(o[0][2 * n2], a, bl[0], bl[1]);
          mma16816(o[0][2 * n2 + 1], a, bl[2], bl[3]);
        }
        if constexpr (DS == 2) {  // O[:, 64:128] += P . v[slot 1]
          uint32_t b1[4];
          ldsm_bt(vst + KV_BYTES, kk, 16 * n2, b1);
          mma16816(o[DS - 1][2 * n2], a, b1[0], b1[1]);
          mma16816(o[DS - 1][2 * n2 + 1], a, b1[2], b1[3]);
        }
      }
    }
    __syncthreads();  // every warp is done with stage s
    if (threadIdx.x == 0 && j + KV_STAGES < nblk) load_kv(j + KV_STAGES);
  }

  // ---- O / l -> ctx
  const size_t pitch = SPLIT ? 2 * (size_t)p.E : (size_t)p.E;  // SPLIT: ctx [M, 2E] = hi | lo
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float lr = quad_sum(l[r]);
    const int t = qt * BLOCK_Q + (int)(qrow + g + 8 * r);
    if (t >= p.T) continue;
    const float inv = lr > 0.f ? 1.0f / lr : 0.f;
    if (p.row_max != nullptr && c == 0) {
      const size_t si = ((size_t)b * p.H + h) * p.T + t;
      p.row_max[si] = m[r] == -INFINITY ? 0.f : m[r];
      p.row_sum[si] = lr;
    }
    __half* dst = p.ctx + ((size_t)(row_base + t) * p.cols + b % p.cols) * pitch + h * HEAD_COLS;
#pragma unroll
    for (int sl = 0; sl < DS; ++sl)
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        const float y0 = o[sl][nb][2 * r] * inv, y1 = o[sl][nb][2 * r + 1] * inv;
        const __half2 h2 = __floats2half2_rn(y0, y1);
        const int col = sl * 64 + nb * 8 + 2 * (int)c;
        *reinterpret_cast<__half2*>(dst + col) = h2;
        if constexpr (SPLIT) {
          const float2 f = __half22float2(h2);
          *reinterpret_cast<__half2*>(dst + p.E + col) = __floats2half2_rn(y0 - f.x, y1 - f.y);
        }
      }
  }
}

template <bool SPLIT, int DS>
inline cudaError_t launch_attention_ds(const CUtensorMap& tmap_q, const CUtensorMap& tmap_kv, const AttnParams& p,
                                       cudaStream_t stream) {
  using namespace attn8_cfg;
  constexpr int smem = smem_bytes((SPLIT || DS == 2) ? 2 : 1);
  auto kern = attention_fwd_kernel<SPLIT, DS>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  const long long total = (long long)p.B * p.H * ((p.T + BLOCK_Q - 1) / BLOCK_Q);
  if (total > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
  return launch_pdl(kern, dim3((unsigned)total), dim3(NUM_THREADS), smem, stream, tmap_q, tmap_kv, p);
}

// fp16 operands in one 64-wide slot run on the warpgroup-MMA kernel (attention_wg.cuh); fp32x3 operands and two-slot
// heads on attention_fwd_kernel above
inline bool attention_fwd_uses_wg(const AttnParams& p) { return p.lo_off == 0 && p.slots == 1; }

// Rows of the K/V TMA box the launched kernel expects (tmap_kv of launch_attention_fwd); the Q box is 128 rows for
// every kernel (and the probability kernels that share the Q map)
inline int attention_fwd_kv_box_rows(const AttnParams& p) {
  return attention_fwd_uses_wg(p) ? attn_wg_cfg::BLOCK_KV : attn8_cfg::BLOCK_KV;
}

inline cudaError_t launch_attention_fwd(const CUtensorMap& tmap_q, const CUtensorMap& tmap_kv, const AttnParams& p,
                                        int num_sms, cudaStream_t stream) {
  if (attention_fwd_uses_wg(p)) return launch_attention_wg(tmap_q, tmap_kv, p, num_sms, stream);
  if (p.lo_off > 0) return launch_attention_ds<true, 1>(tmap_q, tmap_kv, p, stream);
  return launch_attention_ds<false, 2>(tmap_q, tmap_kv, p, stream);
}

}  // namespace esmb200
