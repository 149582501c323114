// esm_b200 — fp8 GEMM: persistent warp-specialised e4m3 wgmma GEMM with block scales (sm_90a), the QKV, fc1 and fc2
// projections of the "fp8" precision.
//
//   out[M, N] = epilogue(sum_kb sa[kb][m] * sb[n / 128][kb] * (A[m, kb] . B[n, kb])), A [M, K] and B [N, K] e4m3,
//   K-major; kb = 128-wide K block.  sa: one scale per row and K block of A, k-block major [ceil(K/128), M]; sb: one
//   scale per 128 x 128 block of B, [ceil(N/128), ceil(K/128)].  Every scale is a power of two (fp8_block_scale).
//   * one CTA per SM walks 128 x 128 output tiles; warpgroup 0: one thread streams K blocks of A and B (128 rows x 128
//     bytes each, one 128B-swizzled row = one scale block) through a 6-stage TMA ring; a partial last K block is
//     zero-filled by TMA on both operands;
//   * warpgroups 1 and 2: rows [0,64) and [64,128) of the tile.  Hopper's fp8 wgmma keeps only about 14 bits in its
//     internal accumulation (DeepSeek-V3 section 3.3.2), so each K block runs 4 x wgmma m64n128k32 into a fresh
//     temporary and is then promoted once, acc += tmp * (sa[row] * sb), in fp32 registers (64 + 64 accumulators per
//     thread; the product of the two power-of-two scales is exact).  The other warpgroup's MMAs run meanwhile;
//   * epilogues (boxes of 64 rows x 128 bytes through shared memory and TMA, as in gemm2.cuh): QKV + RoPE -> fp16 (the
//     box code of gemm2.cuh, epi_qkv_box), bias + residual reduce-add into the fp32 stream, and fc1's bias + erf-GELU
//     -> e4m3 with one scale per row and 128 columns (the A operand of fc2): a row's 128 columns are spread over the 4
//     threads of a quad, so its amax takes two shuffles.
#pragma once

#include "gemm_common.cuh"

namespace esmb200 {

enum : int { EPI_GELU_FP8 = 5 };  // fc1: bias + erf-GELU -> e4m3 [M, N] and its scales [N / 128, M]

struct Fp8GemmParams {
  GemmParams g;     // M, N, K, bias and the QKV fields as for gemm2
  const float* sa;  // [ceil(K/128), M] scales of A
  const float* sb;  // [ceil(N/128), ceil(K/128)] scales of B
  float* so;        // EPI_GELU_FP8: [N/128, M] scales of the e4m3 output
};

namespace gemm_fp8_cfg {
constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 128;
constexpr int BLOCK_K = 128;  // bytes of e4m3: one swizzled row, one scale block
constexpr int STAGES = 6;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K;  // 16 KB
constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K;  // 16 KB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int BOX_ROWS = 128;     // rows of an A or B operand TMA box
constexpr int OUT_BOX_ROWS = 64;  // rows of an output TMA box: one MMA warpgroup's half of the tile
constexpr int OUT_BOX_BYTES = OUT_BOX_ROWS * 128;
constexpr int OUT_BUFS = 2;
constexpr int NUM_THREADS = 384;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * OUT_BUFS * OUT_BOX_BYTES + 1024 + 256;  // 230656 B
// the producer's expect_tx counts one box of BOX_ROWS rows per operand: the tensor maps must use exactly these boxes
static_assert(A_STAGE_BYTES == BOX_ROWS * BLOCK_K && B_STAGE_BYTES == BOX_ROWS * BLOCK_K, "fp8 TMA boxes != stages");
}  // namespace gemm_fp8_cfg

// m64n128k32, e4m3 x e4m3 -> fp32, A and B K-major in shared memory; d[64] in the m64n256k16 fragment layout
__device__ __forceinline__ void wgmma_m64n128k32_e4m3(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void st_shared_u16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}

template <int EPI>
__global__ void __launch_bounds__(gemm_fp8_cfg::NUM_THREADS, 1)
gemm_fp8_e4m3_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     const __grid_constant__ CUtensorMap tmap_o, const Fp8GemmParams fp) {
  using namespace gemm_fp8_cfg;
  const GemmParams& p = fp.g;
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
  const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;

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
  pdl_wait();

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
          mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
          tma_load_2d(smem_a + s * A_STAGE_BYTES, &tmap_a, &full_bar[s], kb * BLOCK_K, m0);
          tma_load_2d(smem_b + s * B_STAGE_BYTES, &tmap_b, &full_bar[s], kb * BLOCK_K, n0);
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
  uint32_t ob = 0;
  uint32_t it = 0;
  float acc[64], tmp[64];

  // gemm2_f16_kernel's store_box: fence, wait for the store two boxes back, warpgroup barrier, one thread issues
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
    const int r0 = m0 + (int)(mw * 64 + warp * 16 + g);  // the thread's rows r0 and r0 + 8
    const float* sb = fp.sb + (size_t)(n0 / BLOCK_N) * num_kb;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const uint32_t s = it % STAGES;
      while (!mbar_try_wait(&full_bar[s], (it / STAGES) & 1)) {
      }
      wgmma_fence();
      const uint64_t da = wgmma_desc_sw128(a_base + s * A_STAGE_BYTES);
      const uint64_t db = wgmma_desc_sw128(b_base + s * B_STAGE_BYTES);
#pragma unroll
      for (int k = 0; k < BLOCK_K / 32; ++k) wgmma_m64n128k32_e4m3(tmp, da + 2 * k, db + 2 * k, k != 0);
      wgmma_commit();
      // the block's scales load under the MMAs; rows >= M (zero-filled by TMA) take scale 0
      const float* sak = fp.sa + (size_t)kb * p.M;
      const float sa0 = r0 < p.M ? __ldg(sak + r0) : 0.f;
      const float sa1 = r0 + 8 < p.M ? __ldg(sak + r0 + 8) : 0.f;
      const float sbk = __ldg(sb + kb);
      wgmma_wait<0>();
      reg_fence_f(tmp);
      if (signal) mbar_arrive(&empty_bar[s]);
      const float f0 = sa0 * sbk, f1 = sa1 * sbk;  // powers of two: exact
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        acc[4 * i] = fmaf(tmp[4 * i], f0, acc[4 * i]);
        acc[4 * i + 1] = fmaf(tmp[4 * i + 1], f0, acc[4 * i + 1]);
        acc[4 * i + 2] = fmaf(tmp[4 * i + 2], f1, acc[4 * i + 2]);
        acc[4 * i + 3] = fmaf(tmp[4 * i + 3], f1, acc[4 * i + 3]);
      }
    }

    // ---- epilogue: thread holds rows r0 and r0 + 8, columns n0 + 8 i + 2 c + {0, 1} for i < 16; TMA clips rows >= M
    const int box_row = m0 + (int)mw * 64;
    if constexpr (EPI == EPI_QKV_ROPE) {  // 64-column fp16 boxes (N % 64 == 0)
#pragma unroll
      for (int gi = 0; gi < 2; ++gi) {
        const int col0 = n0 + gi * 64;
        if (col0 >= p.N) break;
        uint32_t hi[16], lo[16];
        epi_qkv_box<false>(acc + 32 * gi, p, col0, r0, c, hi, lo);
        stage_box_f16(smem_u32(out_bufs + ob * OUT_BOX_BYTES), warp, lane, hi);
        store_box(col0, box_row);
      }
    } else if constexpr (EPI == EPI_BIAS_RESIDUAL) {  // 32-column fp32 boxes, x += y in the L2
#pragma unroll
      for (int gi = 0; gi < 4; ++gi) {
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
          for (int hr = 0; hr < 2; ++hr)
            st_shared_f32x2(sw128(buf, warp * 16 + 8 * hr + g, 2 * b + c / 2) + (c % 2) * 8,
                            acc[4 * i + 2 * hr] + bb.x, acc[4 * i + 2 * hr + 1] + bb.y);
        }
        store_box(col0, box_row);
      }
    } else {  // EPI_GELU_FP8: one 128-column e4m3 box (N % 128 == 0) and one scale per row
      float amax[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * i + 2 * (int)c));
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          acc[4 * i + 2 * hr] = gelu_erf(acc[4 * i + 2 * hr] + bb.x);
          acc[4 * i + 2 * hr + 1] = gelu_erf(acc[4 * i + 2 * hr + 1] + bb.y);
          amax[hr] = fmaxf(amax[hr], fmaxf(fabsf(acc[4 * i + 2 * hr]), fabsf(acc[4 * i + 2 * hr + 1])));
        }
      }
      const uint32_t buf = smem_u32(out_bufs + ob * OUT_BOX_BYTES);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        amax[hr] = fmaxf(amax[hr], __shfl_xor_sync(0xffffffffu, amax[hr], 1));
        amax[hr] = fmaxf(amax[hr], __shfl_xor_sync(0xffffffffu, amax[hr], 2));
        const float sc = fp8_block_scale(amax[hr]), inv = __frcp_rn(sc);  // y * inv == y / sc exactly
        const int row = r0 + 8 * hr;
        if (c == 0 && row < p.M) fp.so[(size_t)(n0 / BLOCK_N) * p.M + row] = sc;
        // bytes 8 i + 2 c ..+1 of the row: 16-byte chunk i / 2, offset 8 (i % 2) + 2 c
#pragma unroll
        for (int i = 0; i < 16; ++i)
          st_shared_u16(sw128(buf, warp * 16 + 8 * hr + g, i / 2) + (i % 2) * 8 + 2 * c,
                        cvt_e4m3x2(acc[4 * i + 2 * hr] * inv, acc[4 * i + 2 * hr + 1] * inv));
      }
      store_box(n0, box_row);
    }
  }
  if (signal) tma_store_wait_all();
}

template <int EPI>
inline cudaError_t launch_gemm_fp8_epi(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to,
                                       const Fp8GemmParams& p, int num_sms, cudaStream_t stream) {
  using namespace gemm_fp8_cfg;
  cudaError_t e =
      cudaFuncSetAttribute(gemm_fp8_e4m3_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
  if (e != cudaSuccess) return e;
  const int tiles = ((p.g.M + BLOCK_M - 1) / BLOCK_M) * ((p.g.N + BLOCK_N - 1) / BLOCK_N);
  const int grid = tiles < num_sms ? tiles : num_sms;
  return launch_pdl(gemm_fp8_e4m3_kernel<EPI>, dim3(grid), dim3(NUM_THREADS), SMEM_BYTES, stream, ta, tb, to, p);
}

}  // namespace esmb200
