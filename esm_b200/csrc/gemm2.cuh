// esm_b200 — GEMM: persistent warp-specialised wgmma GEMM with fused epilogues (sm_90a).
//
//   out[M, N] = epilogue(A[M, K] . B[N, K]^T), A and B fp16 K-major, fp32 accumulation.
//   * one CTA per SM walks 128 x 256 output tiles (tile = m_blk * tiles_n + n_blk, strided over the grid);
//   * warpgroup 0: one thread streams 64-wide K slabs of A (128 rows) and B (256 rows) through a 4-stage TMA ring
//     (48 KB per stage, 128B swizzle) and keeps running ahead into the next tile while the MMA warpgroups finish;
//   * warpgroups 1 and 2: rows [0,64) and [64,128) of the tile, wgmma m64n256k16 straight from the swizzled stages,
//     one slab in flight behind the one being issued; the accumulators (128 fp32 registers per thread) are turned into
//     the output by the epilogue: bias / q-scale + RoPE / erf-GELU in registers, then box by box (64 rows x 128 bytes)
//     into a 128B-swizzled staging buffer in shared memory (stmatrix for fp16, st.shared for fp32), which one thread
//     hands to a TMA store, or for the residual update x += y to a TMA reduce-add performed by the L2 (each element
//     has exactly one writer and one add: bit-reproducible).  Two staging buffers per warpgroup, so the stores drain
//     while the warpgroup fills the next box and runs the next tile's MMAs.
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
constexpr int OUT_BOX_ROWS = 64;  // rows of an output TMA box: one MMA warpgroup's half of the tile
constexpr int OUT_BOX_BYTES = OUT_BOX_ROWS * 128;  // 64 fp16 or 32 fp32 columns per row
constexpr int OUT_BUFS = 2;       // staging buffers per MMA warpgroup
constexpr int NUM_THREADS = 384;  // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * OUT_BUFS * OUT_BOX_BYTES + 1024 + 256;  // 230656 B
}  // namespace gemm2_cfg

// SPLIT ("fp32x3" precision): both operands are stored as fp16 hi | lo halves along K (A [M,2K], B [N,2K]); the K loop
// runs hi*hi + lo*hi + hi*lo (three passes over the same fp32 accumulator: 22 significand bits per operand, the
// dropped lo*lo term is 2^-22 relative), and fp16 outputs are written as hi | lo pairs as well (lo part p.lo_col_off
// columns to the right in an [M, 2N] output map).  Requires K % 64 == 0.
template <int EPI, bool SPLIT = false>
__global__ void __launch_bounds__(gemm2_cfg::NUM_THREADS, 1)
gemm2_f16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_o, const GemmParams p) {
  using namespace gemm2_cfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  uint8_t* smem_out = smem + STAGES * STAGE_BYTES;  // [2 warpgroups][OUT_BUFS] output boxes
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_out + 2 * OUT_BUFS * OUT_BOX_BYTES);
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
    tma_prefetch_desc(&tmap_o);
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
  uint8_t* const out_bufs = smem_out + mw * OUT_BUFS * OUT_BOX_BYTES;
  uint32_t ob = 0;  // staging buffer the warpgroup fills next
  uint32_t it = 0;
  float acc[128];

  // Hand the filled staging buffer to the TMA engine as the output box at (column c0, row c1).  Every thread fences
  // its shared-memory writes for the async proxy; before the warpgroup barrier the issuing thread waits until the
  // previous box's store has finished reading the other buffer, so after the barrier that buffer is free to fill while
  // this box drains (one barrier per box).  Only the issuing thread commits bulk groups, so only it may wait on them.
  auto store_box = [&](int c0, int c1) {
    fence_proxy_async_smem();
    if (signal) tma_store_wait_read<0>();
    named_bar_sync(1 + mw, 128);
    if (signal) {
      if constexpr (EPI == EPI_BIAS_RESIDUAL) {
        tma_reduce_add_2d(&tmap_o, out_bufs + ob * OUT_BOX_BYTES, c0, c1);
      } else {
        tma_store_2d(&tmap_o, out_bufs + ob * OUT_BOX_BYTES, c0, c1);
      }
      tma_store_commit();
    }
    ob ^= 1;
  };

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

    // ---- epilogue: thread holds rows r0 and r0 + 8, columns n0 + 8 i + 2 c + {0, 1} for i < 32.  Boxes whose first
    // column is >= N are skipped (N % 64 == 0 for fp16 outputs, so fp16 boxes are whole); TMA clips rows >= M and the
    // columns >= N of a partial fp32 box.
    const int r0 = m0 + (int)(mw * 64 + warp * 16 + g);
    const int box_row = m0 + (int)mw * 64;
    if constexpr (EPI == EPI_QKV_ROPE || EPI == EPI_BIAS_GELU) {
#pragma unroll
      for (int gi = 0; gi < 4; ++gi) {  // 64-column boxes
        const int col0 = n0 + gi * 64;
        if (col0 >= p.N) break;
        uint32_t hi[16], lo[16];  // [2 b + hr]: 8-column block b of the box, rows r0 + 8 hr
        if constexpr (EPI == EPI_QKV_ROPE) {
          epi_qkv_box<SPLIT>(acc + 32 * gi, p, col0, r0, c, hi, lo);
        } else {
#pragma unroll
          for (int b = 0; b < 8; ++b) {
            const int i = 8 * gi + b;
            const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * b + 2 * (int)c));
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const float y0 = gelu_erf(acc[4 * i + 2 * hr] + bb.x), y1 = gelu_erf(acc[4 * i + 2 * hr + 1] + bb.y);
              hi[2 * b + hr] = pack_half2(y0, y1);
              if constexpr (SPLIT) {
                const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi[2 * b + hr]));
                lo[2 * b + hr] = pack_half2(y0 - f.x, y1 - f.y);
              }
            }
          }
        }
        stage_box_f16(smem_u32(out_bufs + ob * OUT_BOX_BYTES), warp, lane, hi);
        store_box(col0, box_row);
        if constexpr (SPLIT) {  // the lo halves: p.lo_col_off columns to the right in the [M, 2N] output map
          stage_box_f16(smem_u32(out_bufs + ob * OUT_BOX_BYTES), warp, lane, lo);
          store_box(p.lo_col_off + col0, box_row);
        }
      }
    } else {  // fp32 output: 32-column boxes
#pragma unroll
      for (int gi = 0; gi < 8; ++gi) {
        const int col0 = n0 + gi * 32;
        if (col0 >= p.N) break;
        const uint32_t buf = smem_u32(out_bufs + ob * OUT_BOX_BYTES);
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int i = 4 * gi + b;
          // N % 16 == 0: an 8-column block is wholly in or out; the bias of an out-of-range block is never stored
          const float2 bb = col0 + 8 * b < p.N
                                ? __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * b + 2 * (int)c))
                                : make_float2(0.f, 0.f);
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            float y0 = acc[4 * i + 2 * hr] + bb.x, y1 = acc[4 * i + 2 * hr + 1] + bb.y;
            if constexpr (EPI == EPI_BIAS_GELU_F32) {
              y0 = gelu_erf(y0);
              y1 = gelu_erf(y1);
            }
            // bytes 32 b + 8 c of row 16 warp + 8 hr + g: 16-byte chunk 2 b + c / 2; 8 rows x 32 bytes per warp
            // store spread over all 32 banks twice (the minimum two wavefronts)
            st_shared_f32x2(sw128(buf, warp * 16 + 8 * hr + g, 2 * b + c / 2) + (c % 2) * 8, y0, y1);
          }
        }
        store_box(col0, box_row);  // EPI_BIAS_RESIDUAL: x += y in the L2
      }
    }
  }
  if (signal) tma_store_wait_all();  // the staging buffers must outlive the stores reading them
}

template <int EPI, bool SPLIT = false>
inline cudaError_t launch_gemm2_epi(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to,
                                    const GemmParams& p, int num_sms, cudaStream_t stream) {
  using namespace gemm2_cfg;
  cudaError_t e =
      cudaFuncSetAttribute(gemm2_f16_kernel<EPI, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  if (e != cudaSuccess) return e;
  const int tiles = ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N);
  const int grid = tiles < num_sms ? tiles : num_sms;
  return launch_pdl(gemm2_f16_kernel<EPI, SPLIT>, dim3(grid), dim3(NUM_THREADS), SMEM_BYTES, stream, ta, tb, to, p);
}

}  // namespace esmb200
