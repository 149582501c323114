// esm_b200 — attention forward for fp16 operands and 64-wide heads (sm_90a): persistent, warp-specialised flash
// attention on warpgroup MMAs (wgmma).
//
// Replaces esm/multihead_attention.py:357-394 for the fp16, one-slot case (every ESM-2 model up to 3B, ESM-1b/1v and
// the MSA Transformer's column attention).  One CTA per SM walks work items w = (sequence, head, 128-query tile),
// w = blockIdx.x, blockIdx.x + gridDim.x, ...: at any moment the CTAs of the GPU work on ~gridDim.x consecutive items,
// i.e. all query tiles of a few (sequence, head) pairs, so each K/V is read from HBM about once and from L2 after.
//   * warpgroup 0: one thread streams each item's Q tile (two buffers) and its 128-key K and V tiles (4-stage ring,
//     separate full barriers for K and V, one empty barrier per stage) with TMA; it runs ahead into the next items
//     while the consumers finish the current one, so no item pays a load latency up front.
//   * warpgroups 1 and 2: query rows [0, 64) and [64, 128) of the tile.  Per key block j:
//       S_j = Q K_j^T        SS wgmma m64n128k16 from the 128B-swizzled Q and K tiles (both K-major)
//       mask, online softmax with the exact running maximum, P_j = fp16(exp(S_j - m_j)) in registers
//       O  += P_j V_j        RS wgmma m64n64k16: P is the register A operand (the accumulator layout of S is the A
//                            fragment layout), V the MN-major B operand read from the same [keys][64] swizzled tile
//     S_{j+1} and P_j V_j are issued together; the warpgroup waits for S_{j+1} only, and the softmax of block j+1
//     runs while P_j V_j is still on the tensor cores (FA3's intra-warpgroup overlap).  The two warpgroups take
//     turns issuing their MMAs (named-barrier ping-pong), so one's softmax runs under the other's MMAs.
// Exactness as in attention8.cuh: P is rounded to fp16 relative to the running maximum (values <= 1), row sums and O
// are fp32; the result depends only on the inputs (fixed order of every sum).
#pragma once

#include "attention_common.cuh"

namespace esmb200 {

namespace attn_wg_cfg {
constexpr int BLOCK_Q = 128;           // query rows per work item: one 64-row half per consumer warpgroup
constexpr int BLOCK_KV = 128;          // keys per K / V tile (the n of the S wgmma)
constexpr int STAGES = 4;              // K/V ring depth
constexpr int Q_BUFS = 2;              // the next item's Q loads while the current item runs
constexpr int TILE_BYTES = 128 * 128;  // 16 KB: 128 rows x 64 fp16 (Q, K and V tiles alike)
constexpr int NUM_THREADS = 384;       // warpgroup 0: TMA producer, warpgroups 1-2: MMA + softmax
constexpr int SMEM_BYTES = (Q_BUFS + 2 * STAGES) * TILE_BYTES + 1024 + 256;  // 165120 B
}  // namespace attn_wg_cfg

__global__ void __launch_bounds__(attn_wg_cfg::NUM_THREADS, 1)
attention_wg_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv,
                    const AttnParams p) {
  using namespace attn_wg_cfg;
  constexpr float LOG2E = attn_cfg::LOG2E;
  constexpr int D = attn_cfg::HEAD_DIM;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;                             // [Q_BUFS]
  uint8_t* smem_k = smem + Q_BUFS * TILE_BYTES;       // [STAGES]
  uint8_t* smem_v = smem_k + STAGES * TILE_BYTES;     // [STAGES]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_v + STAGES * TILE_BYTES);
  uint64_t* q_full = bars;                 // [Q_BUFS] TMA -> consumers
  uint64_t* q_empty = bars + Q_BUFS;       // [Q_BUFS] consumers (one arrival per warpgroup) -> TMA
  uint64_t* k_full = bars + 2 * Q_BUFS;    // [STAGES]
  uint64_t* v_full = k_full + STAGES;      // [STAGES]
  uint64_t* kv_empty = v_full + STAGES;    // [STAGES] one arrival per consumer warpgroup

  const uint32_t wg = __shfl_sync(0xffffffffu, threadIdx.x / 128, 0);
  const int nqt = (p.T + BLOCK_Q - 1) / BLOCK_Q;
  const int items = p.B * p.H * nqt;  // the launcher checks that this fits an int

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_kv);
    for (int i = 0; i < Q_BUFS; ++i) {
      mbar_init(&q_full[i], 1);
      mbar_init(&q_empty[i], 2);
    }
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&kv_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // everything below reads the previous kernel's output (qkv, key bits) or writes ctx

  // Both roles walk the same items and skip the same ones (kvlen == 0: no loads, zero context), so the Q buffer and
  // ring counters (qi, it) advance identically on both sides.
  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<24>();
    if (threadIdx.x == 0) {
      auto wait_empty = [](uint64_t* bar, uint32_t parity) {
#if ESMB200_WATCHDOG
        uint32_t polls = 0;
        while (!mbar_try_wait(bar, parity)) {
          __nanosleep(64);
          if (++polls == (1u << 24)) __trap();
        }
#else
        while (!mbar_try_wait(bar, parity)) __nanosleep(64);
#endif
      };
      uint32_t qi = 0, it = 0;
      for (int w = blockIdx.x; w < items; w += gridDim.x) {
        const int qt = w % nqt, h = (w / nqt) % p.H, b = w / (nqt * p.H);
        const int nblk = (__ldg(p.kvlen + b) + BLOCK_KV - 1) / BLOCK_KV;
        if (nblk == 0) continue;
        const int row_base = (b / p.cols) * p.T;
        const int x0 = (b % p.cols) * 3 * p.E + h * D;
        const uint32_t qb = qi % Q_BUFS;
        wait_empty(&q_empty[qb], ((qi / Q_BUFS) & 1) ^ 1);
        mbar_arrive_expect_tx(&q_full[qb], TILE_BYTES);
        tma_load_2d(smem_q + qb * TILE_BYTES, &tmap_q, &q_full[qb], x0, row_base + qt * BLOCK_Q);
        ++qi;
        for (int j = 0; j < nblk; ++j, ++it) {
          const uint32_t s = it % STAGES;
          wait_empty(&kv_empty[s], ((it / STAGES) & 1) ^ 1);
          mbar_arrive_expect_tx(&k_full[s], TILE_BYTES);
          tma_load_2d(smem_k + s * TILE_BYTES, &tmap_kv, &k_full[s], x0 + p.E, row_base + j * BLOCK_KV);
          mbar_arrive_expect_tx(&v_full[s], TILE_BYTES);
          tma_load_2d(smem_v + s * TILE_BYTES, &tmap_kv, &v_full[s], x0 + 2 * p.E, row_base + j * BLOCK_KV);
        }
      }
    }
    return;
  }

  // ===================== MMA + softmax warpgroups =====================
  setmaxnreg_inc<240>();
  const uint32_t mw = wg - 1;                    // rows [64 mw, 64 mw + 64) of the item's query tile
  const uint32_t warp = (threadIdx.x / 32) % 4;  // rows [16 warp, +16) of the warpgroup's 64
  const uint32_t lane = threadIdx.x % 32, g = lane / 4, c = lane % 4;
  const bool signal = (threadIdx.x % 128) == 0;
  const uint32_t q_base = smem_u32(smem_q) + mw * 64 * 128;
  const uint32_t k_base = smem_u32(smem_k), v_base = smem_u32(smem_v);
  uint32_t qi = 0, it = 0;

  // Ping-pong between the two warpgroups (FA3's inter-warpgroup schedule): a warpgroup issues its MMAs only on its
  // turn (named barrier 1 + mw) and hands the turn to the other one right after, so one warpgroup's softmax runs
  // while the other's MMAs occupy the tensor cores.  Both warpgroups take the same number of turns (nblk + 1 per
  // item); warpgroup 2 starts by giving warpgroup 1 the first turn.
  auto turn_begin = [&]() { named_bar_sync(1 + mw, 256); };
  auto turn_end = [&]() { named_bar_arrive(2 - mw, 256); };
  if (mw == 1) turn_end();

  // no mbar_wait in this kernel: the watchdog's printf is a function call, and any call in a wgmma kernel makes ptxas
  // serialise every wgmma (C7510); a lost arrival traps without the message instead
  auto wait_full = [](uint64_t* bar, uint32_t parity) {
#if ESMB200_WATCHDOG
    uint32_t polls = 0;
    while (!mbar_try_wait(bar, parity))
      if (++polls == (1u << 26)) __trap();
#else
    while (!mbar_try_wait(bar, parity)) {
    }
#endif
  };

  for (int w = blockIdx.x; w < items; w += gridDim.x) {
    const int qt = w % nqt, h = (w / nqt) % p.H, b = w / (nqt * p.H);
    const int nblk = (__ldg(p.kvlen + b) + BLOCK_KV - 1) / BLOCK_KV;
    const uint32_t* kb_ptr = p.keybits + (size_t)b * p.words;
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

    if (nblk > 0) {
      const uint32_t qb = qi % Q_BUFS;
      const uint64_t dq = wgmma_desc_sw128(q_base + qb * TILE_BYTES);
      float sc[64];     // S of the block in flight, then exp(S - m) of that block in fp32
      uint32_t pa[32];  // fp16 P of the block whose P.V is in flight: pa[2 i + r] = columns 8i + 2c.. of row g + 8 r
      float alpha[2];   // factor taking O and l from the previous running maximum to the current one

      // S = Q K^T of block j into sc (asynchronous: committed, not waited for)
      auto issue_qk = [&](uint32_t s) {
        const uint64_t dk = wgmma_desc_sw128(k_base + s * TILE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < D / 16; ++k) wgmma_m64n128k16(sc, dq + 2 * k, dk + 2 * k, k);
        wgmma_commit();
      };
      // O = alpha O + P V of the block in stage s with P in pa (asynchronous)
      auto issue_pv = [&](uint32_t s) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
          o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
        }
        wgmma_fence();
        const uint64_t dv = wgmma_desc_sw128_mn(v_base + s * TILE_BYTES);
#pragma unroll
        for (int kk = 0; kk < BLOCK_KV / 16; ++kk) {
          const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
          wgmma_m64n64k16_rs(o, a, dv + kk * (2048 >> 4));
        }
        wgmma_commit();
      };
      // key-padding mask, running maximum and sum of block j: sc -> exp(sc - m) (fp32), alpha
      auto softmax = [&](int j) {
        const uint4 kw = __ldg(reinterpret_cast<const uint4*>(kb_ptr + 4 * j));
        if ((kw.x & kw.y & kw.z & kw.w) != 0xffffffffu) {  // uniform over the CTA: most blocks have no padded key
          const uint32_t wd[4] = {kw.x, kw.y, kw.z, kw.w};
#pragma unroll
          for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (!((wd[i / 4] >> ((i % 4) * 8 + 2 * c + e)) & 1u)) sc[4 * i + e] = sc[4 * i + 2 + e] = -INFINITY;
        }
        // Tree reductions (max here, four partial sums below): two warps per SM sub-partition run the softmax, too
        // few to hide 32-long chains of dependent operations.
        float mx[2][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int r = 0; r < 2; ++r)
            mx[r][i] = fmaxf(fmaxf(sc[4 * i + 2 * r], sc[4 * i + 2 * r + 1]),
                             fmaxf(sc[4 * (i + 8) + 2 * r], sc[4 * (i + 8) + 2 * r + 1]));
#pragma unroll
        for (int w = 4; w >= 1; w /= 2)
#pragma unroll
          for (int i = 0; i < w; ++i) {
            mx[0][i] = fmaxf(mx[0][i], mx[0][i + w]);
            mx[1][i] = fmaxf(mx[1][i], mx[1][i + w]);
          }
        float ref[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float mn = fmaxf(m[r], quad_max(mx[r][0]));
          alpha[r] = (mn == -INFINITY) ? 1.f : ex2_approx((m[r] - mn) * LOG2E);  // ex2(-inf) = 0 before the first key
          m[r] = mn;
          ref[r] = (mn == -INFINITY) ? 0.f : -mn * LOG2E;
          l[r] *= alpha[r];
        }
        float ls[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            sc[4 * i + 2 * r] = ex2_approx(fmaf(sc[4 * i + 2 * r], LOG2E, ref[r]));
            sc[4 * i + 2 * r + 1] = ex2_approx(fmaf(sc[4 * i + 2 * r + 1], LOG2E, ref[r]));
            ls[r][i % 4] += sc[4 * i + 2 * r] + sc[4 * i + 2 * r + 1];
          }
#pragma unroll
        for (int r = 0; r < 2; ++r) l[r] += (ls[r][0] + ls[r][1]) + (ls[r][2] + ls[r][3]);
      };
      // P = fp16(sc), once the previous P.V no longer reads pa
      auto convert_p = [&]() {
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int r = 0; r < 2; ++r) pa[2 * i + r] = pack_half2(sc[4 * i + 2 * r], sc[4 * i + 2 * r + 1]);
      };

      wait_full(&q_full[qb], (qi / Q_BUFS) & 1);
      ++qi;
      uint32_t s = it % STAGES;
      wait_full(&k_full[s], (it / STAGES) & 1);
      turn_begin();
      issue_qk(s);
      turn_end();
      wgmma_wait<0>();
      reg_fence_f(sc);
      if (nblk == 1 && signal) mbar_arrive(&q_empty[qb]);
      softmax(0);
      convert_p();
      wait_full(&v_full[s], (it / STAGES) & 1);
      for (int j = 1; j < nblk; ++j) {
        const uint32_t sp = s;  // stage of block j - 1 (its V has arrived)
        ++it;
        s = it % STAGES;
        wait_full(&k_full[s], (it / STAGES) & 1);
        turn_begin();
        issue_qk(s);
        issue_pv(sp);     // O = alpha_{j-1} O + P_{j-1} V_{j-1}
        turn_end();
        wgmma_wait<1>();  // S_j is ready; P_{j-1} V_{j-1} may still run
        reg_fence_f(sc);
        if (j == nblk - 1 && signal) mbar_arrive(&q_empty[qb]);
        softmax(j);
        // V_j, needed by the next P.V, is waited for here rather than before that issue: its spin loop ends the
        // basic block of the softmax.  ptxas schedules a wgmma wait as early as its basic block allows; in the same
        // block as the softmax the wait below would move in front of the exponentials and serialise them behind
        // P_{j-1} V_{j-1}.
        wait_full(&v_full[s], (it / STAGES) & 1);
        wgmma_wait<0>();
        reg_fence_f(o);
        reg_fence_f(sc);  // keeps the conversion after the wait (pa itself is guarded by ptxas's wgmma tracking)
        if (signal) mbar_arrive(&kv_empty[sp]);
        convert_p();
      }
      turn_begin();
      issue_pv(s);
      turn_end();
      wgmma_wait<0>();
      reg_fence_f(o);
      if (signal) mbar_arrive(&kv_empty[s]);
      ++it;
    }

    // ---- O / l -> ctx (kvlen == 0: O = 0, l = 0 -> zero context and zero statistics)
    const int row_base = (b / p.cols) * p.T;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float lr = quad_sum(l[r]);
      const int t = qt * BLOCK_Q + (int)(mw * 64 + warp * 16 + g + 8 * r);
      if (t >= p.T) continue;
      const float inv = lr > 0.f ? 1.0f / lr : 0.f;
      if (p.row_max != nullptr && c == 0) {
        const size_t si = ((size_t)b * p.H + h) * p.T + t;
        p.row_max[si] = m[r] == -INFINITY ? 0.f : m[r];
        p.row_sum[si] = lr;
      }
      __half* dst = p.ctx + ((size_t)(row_base + t) * p.cols + b % p.cols) * p.E + h * D;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<__half2*>(dst + i * 8 + 2 * (int)c) =
            __floats2half2_rn(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
    }
  }
  if (mw == 0) turn_begin();  // take warpgroup 2's last hand-off: no arrival is left pending on barrier 1
}

inline cudaError_t launch_attention_wg(const CUtensorMap& tmap_q, const CUtensorMap& tmap_kv, const AttnParams& p,
                                       int num_sms, cudaStream_t stream) {
  using namespace attn_wg_cfg;
  cudaError_t e = cudaFuncSetAttribute(attention_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  if (e != cudaSuccess) return e;
  const long long items = (long long)p.B * p.H * ((p.T + BLOCK_Q - 1) / BLOCK_Q);
  if (items > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
  const int grid = items < num_sms ? (int)items : num_sms;
  return launch_pdl(attention_wg_kernel, dim3(grid), dim3(NUM_THREADS), SMEM_BYTES, stream, tmap_q, tmap_kv, p);
}

}  // namespace esmb200
