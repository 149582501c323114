// esm_b200 — GEMM: persistent warp-specialised wgmma GEMM with fused epilogues (sm_90a).
//
//   out[M, N] = epilogue(A[M, K] . B[N, K]^T), A and B fp16 K-major, fp32 accumulation.
//   * one CTA per SM walks 128 x 256 output tiles (tile = m_blk * tiles_n + n_blk, strided over the grid);
//   * warpgroup 0: one thread streams 64-wide K slabs of A (128 rows) and B (256 rows) through a 4-stage TMA ring
//     (48 KB per stage, 128B swizzle) and keeps running ahead into the next tile while the MMA warpgroups finish;
//   * warpgroups 1 and 2: rows [0,64) and [64,128) of the tile, wgmma m64n256k16 straight from the swizzled stages,
//     one slab in flight behind the one being issued; the accumulators (128 fp32 registers per thread) are turned into
//     the output by the epilogue in registers: bias / q-scale + RoPE / erf-GELU, fp16 or fp32 stores, or the
//     residual update x += y (each element has exactly one writer: no atomics, bit-reproducible).
#pragma once

#include "gemm_common.cuh"

namespace esmb200 {

namespace gemm2_cfg {
constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 256;
constexpr int HALF_N = 128;   // B rows per TMA box (two boxes per stage)
constexpr int BLOCK_K = 64;
constexpr int STAGES = 4;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;  // 32 KB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int BOX_M = 128;        // rows of an A-operand TMA box
constexpr int NUM_THREADS = 384;  // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
}  // namespace gemm2_cfg

// SPLIT ("fp32x3" precision): both operands are stored as fp16 hi | lo halves along K (A [M,2K], B [N,2K]); the K loop
// runs hi*hi + lo*hi + hi*lo (three passes over the same fp32 accumulator: 22 significand bits per operand, the
// dropped lo*lo term is 2^-22 relative), and fp16 outputs are written as hi | lo pairs as well (lo part p.lo_col_off
// columns to the right, row pitch 2 * ldo).  Requires K % 64 == 0.
template <int EPI, bool SPLIT = false>
__global__ void __launch_bounds__(gemm2_cfg::NUM_THREADS, 1)
gemm2_f16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const GemmParams p) {
  using namespace gemm2_cfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full_bar = bars;            // [STAGES] TMA -> MMA
  uint64_t* empty_bar = bars + STAGES;  // [STAGES] MMA warpgroups -> TMA (one arrival each)

  const uint32_t wg = __shfl_sync(0xffffffffu, threadIdx.x / 128, 0);
  const int tiles_m = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int tiles_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb1 = (p.K + BLOCK_K - 1) / BLOCK_K;  // a partial last K slab is zero-filled by TMA on both operands
  const int num_kb = SPLIT ? 3 * num_kb1 : num_kb1;   // SPLIT: slab kb/3, operand halves by kb%3

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // A (and x for the residual update) come from the previous kernel on the stream

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * BLOCK_M, n0 = (tile % tiles_n) * BLOCK_N;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const uint32_t s = it % STAGES;
          while (!mbar_try_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1)) __nanosleep(64);
          int a_col = kb * BLOCK_K, b_col = kb * BLOCK_K;
          if constexpr (SPLIT) {
            const int part = kb % 3;  // 0: hi*hi, 1: lo*hi, 2: hi*lo
            a_col = (kb / 3) * BLOCK_K + (part == 1 ? p.K : 0);
            b_col = (kb / 3) * BLOCK_K + (part == 2 ? p.K : 0);
          }
          mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
          tma_load_2d(smem_a + s * A_STAGE_BYTES, &tmap_a, &full_bar[s], a_col, m0);
          tma_load_2d(smem_b + s * B_STAGE_BYTES, &tmap_b, &full_bar[s], b_col, n0);
          tma_load_2d(smem_b + s * B_STAGE_BYTES + HALF_N * 128, &tmap_b, &full_bar[s], b_col, n0 + HALF_N);
        }
      }
    }
    return;
  }

  // ===================== MMA + epilogue warpgroups =====================
  setmaxnreg_inc<232>();
  const uint32_t mw = wg - 1;                    // rows [64 mw, 64 mw + 64) of the tile
  const uint32_t warp = (threadIdx.x / 32) % 4;  // rows [16 warp, +16) of the warpgroup's 64
  const uint32_t lane = threadIdx.x % 32;
  const uint32_t g = lane / 4, c = lane % 4;
  const bool signal = (threadIdx.x % 128) == 0;
  const uint32_t a_base = smem_u32(smem_a) + mw * 64 * 128;
  const uint32_t b_base = smem_u32(smem_b);
  const size_t pitch = (SPLIT && (EPI == EPI_QKV_ROPE || EPI == EPI_BIAS_GELU)) ? 2 * (size_t)p.ldo : (size_t)p.ldo;
  uint32_t it = 0;
  float acc[128];

  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = (tile / tiles_n) * BLOCK_M, n0 = (tile % tiles_n) * BLOCK_N;
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const uint32_t s = it % STAGES;
      // plain try_wait loops in this kernel: the watchdog's printf is a function call, and any call in a wgmma kernel
      // makes ptxas serialise every wgmma (C7510)
      while (!mbar_try_wait(&full_bar[s], (it / STAGES) & 1)) {
      }
      wgmma_fence();
      const uint64_t da = wgmma_desc_sw128(a_base + s * A_STAGE_BYTES);
      const uint64_t db = wgmma_desc_sw128(b_base + s * B_STAGE_BYTES);
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) wgmma_m64n256k16(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();  // the previous slab's MMAs have read their stage
      if (kb > 0 && signal) mbar_arrive(&empty_bar[(it + STAGES - 1) % STAGES]);
    }
    wgmma_wait<0>();
    reg_fence_f(acc);
    if (signal) mbar_arrive(&empty_bar[(it + STAGES - 1) % STAGES]);

    // ---- epilogue: thread holds rows r0 and r0 + 8, columns n0 + 8 i + 2 c + {0, 1} for i < 32
    const int r0 = m0 + (int)(mw * 64 + warp * 16 + g);
    const int rows[2] = {r0, r0 + 8};
    if constexpr (EPI == EPI_QKV_ROPE) {
      const bool rope = p.rope_cos != nullptr;
      const int ld = p.rope_ld == 64 ? 64 : 32;
#pragma unroll
      for (int gi = 0; gi < 4; ++gi) {  // 64-column groups: column j pairs with j + 32 (same thread)
        const int col0 = n0 + gi * 64;
        if (col0 >= p.N) break;
        const int sect = col0 / p.E;  // 0 q, 1 k, 2 v
        const float sc = (sect == 0) ? p.q_scale : 1.0f;
        const int slot = p.rope_ld == 64 ? ((col0 >> 6) & 1) : 0;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int row = rows[hr];
          if (row >= p.M) continue;
          const int t = row % p.T;
          __half* o = reinterpret_cast<__half*>(p.out) + (size_t)row * pitch;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int j = 8 * q + 2 * (int)c;  // column pair (j, j + 1) and (j + 32, j + 33) of the group
            const float2 bl = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + j));
            const float2 bh = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 32 + j));
            float a0 = (acc[4 * (8 * gi + q) + 2 * hr] + bl.x) * sc, a1 = (acc[4 * (8 * gi + q) + 2 * hr + 1] + bl.y) * sc;
            float b0 = (acc[4 * (8 * gi + q + 4) + 2 * hr] + bh.x) * sc;
            float b1 = (acc[4 * (8 * gi + q + 4) + 2 * hr + 1] + bh.y) * sc;
            if (sect < 2 && rope) {  // rotary_embedding.py:16-20, rotate_half = cat(-x2, x1)
              const float2 cs = __ldg(reinterpret_cast<const float2*>(p.rope_cos + (size_t)t * ld + slot * 32 + j));
              const float2 sn = __ldg(reinterpret_cast<const float2*>(p.rope_sin + (size_t)t * ld + slot * 32 + j));
              const float ra0 = a0 * cs.x - b0 * sn.x, rb0 = b0 * cs.x + a0 * sn.x;
              const float ra1 = a1 * cs.y - b1 * sn.y, rb1 = b1 * cs.y + a1 * sn.y;
              a0 = ra0; b0 = rb0; a1 = ra1; b1 = rb1;
            }
            const __half2 ha = __floats2half2_rn(a0, a1), hb = __floats2half2_rn(b0, b1);
            *reinterpret_cast<__half2*>(o + col0 + j) = ha;
            *reinterpret_cast<__half2*>(o + col0 + 32 + j) = hb;
            if constexpr (SPLIT) {
              const float2 fa = __half22float2(ha), fb = __half22float2(hb);
              *reinterpret_cast<__half2*>(o + p.lo_col_off + col0 + j) = __floats2half2_rn(a0 - fa.x, a1 - fa.y);
              *reinterpret_cast<__half2*>(o + p.lo_col_off + col0 + 32 + j) = __floats2half2_rn(b0 - fb.x, b1 - fb.y);
            }
          }
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = n0 + 8 * i + 2 * (int)c;
        if (col >= p.N) break;  // N % 32 == 0 (fp32) / % 64 == 0 (fp16): whole 8-column blocks are in or out
        const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int row = rows[hr];
          if (row >= p.M) continue;
          float y0 = acc[4 * i + 2 * hr] + bb.x, y1 = acc[4 * i + 2 * hr + 1] + bb.y;
          if constexpr (EPI == EPI_BIAS_GELU || EPI == EPI_BIAS_GELU_F32) {
            y0 = gelu_erf(y0);
            y1 = gelu_erf(y1);
          }
          if constexpr (EPI == EPI_BIAS_GELU) {
            __half* o = reinterpret_cast<__half*>(p.out) + (size_t)row * pitch + col;
            const __half2 h = __floats2half2_rn(y0, y1);
            *reinterpret_cast<__half2*>(o) = h;
            if constexpr (SPLIT) {
              const float2 f = __half22float2(h);
              *reinterpret_cast<__half2*>(o + p.lo_col_off) = __floats2half2_rn(y0 - f.x, y1 - f.y);
            }
          } else {
            float2* o = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + (size_t)row * pitch + col);
            if constexpr (EPI == EPI_BIAS_RESIDUAL) {
              const float2 x = *o;
              *o = make_float2(x.x + y0, x.y + y1);
            } else {
              *o = make_float2(y0, y1);
            }
          }
        }
      }
    }
  }
}

template <int EPI, bool SPLIT = false>
inline cudaError_t launch_gemm2_epi(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int num_sms,
                                    cudaStream_t stream) {
  using namespace gemm2_cfg;
  cudaError_t e =
      cudaFuncSetAttribute(gemm2_f16_kernel<EPI, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  if (e != cudaSuccess) return e;
  const int tiles = ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N);
  const int grid = tiles < num_sms ? tiles : num_sms;
  return launch_pdl(gemm2_f16_kernel<EPI, SPLIT>, dim3(grid), dim3(NUM_THREADS), SMEM_BYTES, stream, ta, tb, p);
}

}  // namespace esmb200
