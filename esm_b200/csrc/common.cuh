// esm_b200 — shared device-side primitives for the sm_90a (Hopper) kernels.
//
// Thin inline-PTX wrappers for the Hopper programming model used by every kernel in this directory: mbarrier
// (transaction barriers), TMA bulk-tensor loads / stores / reduce-adds, wgmma (warpgroup MMA from shared-memory
// descriptors), warp-level mma.sync + ldmatrix on 128B-swizzled TMA tiles.
// No CUTLASS/CuTe dependency: everything is spelled out so `cuobjdump -sass` maps 1:1 to source.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#ifndef ESMB200_WATCHDOG
#define ESMB200_WATCHDOG 1   // trap instead of hanging forever on a lost mbarrier arrival
#endif

namespace esmb200 {

constexpr uint32_t kWarp = 32;

// ---------------------------------------------------------------------------------------------
// address helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(r));
  return r;
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "elect.sync _|P1, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

// make barrier inits visible to the async proxy (TMA)
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// Blocking wait on phase `parity`. try_wait suspends in hardware for a bounded time (~100 clk), so this is not a
// hot spin. With the watchdog on, a lost arrival traps after 2^26 polls (a few seconds) instead of hanging the box;
// the poll counter costs one integer add + compare per iteration.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
#if ESMB200_WATCHDOG
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++polls == (1u << 26)) {
      printf("esmb200: mbarrier watchdog block=(%d,%d,%d) thread=%d bar=%u parity=%u\n", blockIdx.x, blockIdx.y,
             blockIdx.z, threadIdx.x, smem_u32(bar), parity);
      __trap();
    }
  }
#else
  while (!mbar_try_wait(bar, parity)) {
  }
#endif
}


// Wait used by producer threads that run far ahead of their consumers (TMA rings): back off between polls so the
// polling thread does not take issue slots from the compute warps sharing its SM sub-partition.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
#if ESMB200_WATCHDOG
  uint32_t polls = 0;
#endif
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(200);
#if ESMB200_WATCHDOG
    if (++polls == (1u << 24)) {
      printf("esmb200: mbarrier watchdog (relaxed) block=(%d,%d,%d) thread=%d bar=%u parity=%u\n", blockIdx.x, blockIdx.y,
             blockIdx.z, threadIdx.x, smem_u32(bar), parity);
      __trap();
    }
#endif
  }
}

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — 2D tile load global -> shared, completion on an mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// Forms taking shared-memory byte addresses (callers keep them in uniform registers: warp-convergent issue loops)
__device__ __forceinline__ void tma_load_2d_addr(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar, int32_t c0,
                                                 int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_addr(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

// L2 eviction-priority variant (policy created with createpolicy)
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0,
                                                 int32_t c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, "
      "%4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "l"(policy)
      : "memory");
}

__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// ---------------------------------------------------------------------------------------------
// warp-level tensor-core MMA (mma.sync m16n8k16, fp16 in / fp32 accumulate) and ldmatrix
// Fragment layouts (PTX ISA "Matrix fragments for mma.m16n8k16"), g = lane / 4, c = lane % 4:
//   A (16x16): a0 = (g, 2c..2c+1)  a1 = (g+8, 2c..)  a2 = (g, 8+2c..)  a3 = (g+8, 8+2c..)
//   B (16x8):  b0 = (k 2c..2c+1, n g)  b1 = (k 8+2c.., n g)
//   C (16x8):  c0,c1 = (g, 2c..2c+1)  c2,c3 = (g+8, 2c..2c+1)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

// stmatrix: the inverse of ldsm_x4 — thread l supplies the address of row l % 8 of matrix l / 8, and r[j] holds
// (row lane / 4, columns 2 (lane % 4) ..+1) of matrix j, which is the mma / wgmma accumulator fragment layout
__device__ __forceinline__ void stsm_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}
__device__ __forceinline__ void st_shared_f32x2(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// byte address of 16-byte chunk `chunk` (0..7) of row `row` in a tile of 128-byte rows written by a TMA box with
// CU_TENSOR_MAP_SWIZZLE_128B (tile base 1024-byte aligned): the chunk index is XORed with row % 8
__device__ __forceinline__ uint32_t sw128(uint32_t base, uint32_t row, uint32_t chunk) {
  return base + row * 128u + ((chunk ^ (row & 7u)) << 4);
}

// A fragment of the 16 x 16 block (rows r0.., K columns 16*kk..) of a K-major SW128 tile
__device__ __forceinline__ void ldsm_a(uint32_t base, uint32_t r0, uint32_t kk, uint32_t (&a)[4]) {
  const uint32_t l = lane_id();
  ldsm_x4(sw128(base, r0 + (l & 15u), 2u * kk + (l >> 4)), a);
}
// B fragments of two n8 blocks (rows n0..n0+15 of a K-major SW128 tile, K columns 16*kk..): b[0..1] block n0, b[2..3] n0+8
__device__ __forceinline__ void ldsm_b(uint32_t base, uint32_t n0, uint32_t kk, uint32_t (&b)[4]) {
  const uint32_t l = lane_id();
  ldsm_x4(sw128(base, n0 + (l & 7u) + ((l >> 4) << 3), 2u * kk + ((l >> 3) & 1u)), b);
}
// B fragments of two n8 blocks from an MN-major SW128 tile (rows = K index, 64 N-elements per row; V in P.V):
// K rows 16*kk.., N columns n0..n0+15: b[0..1] block n0, b[2..3] block n0+8
__device__ __forceinline__ void ldsm_bt(uint32_t base, uint32_t kk, uint32_t n0, uint32_t (&b)[4]) {
  const uint32_t l = lane_id();
  ldsm_x4_t(sw128(base, 16u * kk + (l & 15u), n0 / 8u + (l >> 4)), b);
}

// ---------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a): D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory
// ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major 128B-swizzled tile with 128-byte rows (64 fp16), as written by a TMA box
// {64, rows} with CU_TENSOR_MAP_SWIZZLE_128B:  bits [0,14) address >> 4, [16,30) LBO >> 4 (unused for swizzled K-major),
// [32,46) SBO >> 4 = 1024 B between 8-row groups, [62,64) layout 1 = SWIZZLE_128B.  A 16-element K step is +32 bytes.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void reg_fence_f(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// m64n256k16, fp16 x fp16 -> fp32; d[128] per thread: d[4*i + 0..1] = (row w*16 + g, col 8i + 2c..), d[4*i + 2..3] = row + 8
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d));
}

// Shared-memory matrix descriptor of an MN-major 128B-swizzled B operand (used with imm-trans-b = 1): rows are the K
// index, each a 128-byte row of 64 fp16 N-elements, as written by a TMA box {64, rows} with CU_TENSOR_MAP_SWIZZLE_128B
// (e.g. V [keys][64] in O += P.V).  The swizzle atom is the same 8 rows x 128 bytes as in the K-major case; SBO = 1024 B
// is the distance between 8-row groups along K, LBO the distance between 64-element atoms along N.  An N extent of 64
// is exactly one atom, so LBO is never applied; it is set to the same 1024 B.  A 16-row K step is +2048 bytes.
__device__ __forceinline__ uint64_t wgmma_desc_sw128_mn(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1024 >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// m64n128k16, fp16 x fp16 -> fp32, A and B K-major in shared memory; d[64] per thread in the m64n256k16 layout:
// d[4*i + 0..1] = (row w*16 + g, col 8i + 2c..), d[4*i + 2..3] = row + 8
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n}\n"
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

// m64n64k16, fp16 x fp16 -> fp32 with A from registers and B an MN-major shared-memory tile (imm-trans-b = 1).
// a[0..3] is the mma.m16n8k16 A fragment of the warp's 16 rows (a0 = (g, 2c..), a1 = (g+8, 2c..), a2 = (g, 8+2c..),
// a3 = (g+8, 8+2c..)), which is the fp16 packing of an fp32 accumulator's columns 16k.. (d[8k + 0..7]).  d[32] as above.
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

// register budget hand-off between warpgroups (producer gives registers to the MMA warpgroups)
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ---------------------------------------------------------------------------------------------
// TMA stores (shared -> global), bulk async-groups
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
// global[tile] += smem[tile] (fp32), performed by the L2 — the residual add without reading x into the SM
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* map, const void* smem_src, int32_t c0,
                                                  int32_t c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute may
// start while its predecessor on the stream is still draining; everything it does before pdl_wait() (barrier init,
// tensor-map prefetch) overlaps the predecessor's tail.  pdl_wait() returns when the predecessor has
// completed and its memory is visible; both instructions are no-ops in a normal launch.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// process-wide switch: -1 = not read yet (environment ESMB200_PDL, default OFF); esmb200_set_option("pdl", v) overrides.
// Kept as an option, off by default.
inline int& pdl_flag() {
  static int flag = -1;
  return flag;
}
inline bool pdl_enabled() {
  int& f = pdl_flag();
  if (f < 0) {
    const char* e = getenv("ESMB200_PDL");
    f = (e && e[0] == '1') ? 1 : 0;
  }
  return f != 0;
}

// host: launch `kernel` with the PDL attribute (ESMB200_PDL=0 disables it)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// ---------------------------------------------------------------------------------------------
// small math helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// fp32 pair helpers (two independent scalar operations; kept as pairs so the callers read like the math)
__device__ __forceinline__ void fma2(float& d0, float& d1, float a0, float a1, float b0, float b1, float c0, float c1) {
  d0 = fmaf(a0, b0, c0);
  d1 = fmaf(a1, b1, c1);
}
__device__ __forceinline__ void add2(float& d0, float& d1, float a0, float a1, float b0, float b1) {
  d0 = a0 + b0;
  d1 = a1 + b1;
}
__device__ __forceinline__ void mul2(float& d0, float& d1, float a0, float a1, float b0, float b1) {
  d0 = a0 * b0;
  d1 = a1 * b1;
}

// 2^x, MUFU.EX2 (max rel. error 2^-22; ex2(-inf) = +0)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------
// fp8 (e4m3) block scaling: q = e4m3(x / s) with s a power of two per block, so x / s and q * s are exact
// ---------------------------------------------------------------------------------------------
// The smallest power of two s with amax / s <= 448 (e4m3's largest finite value), from the exponent bits: amax = m 2^e
// with m in [1, 2) needs s = 2^(e - 8) when m <= 1.75 (448 = 1.75 * 2^8), else 2^(e - 7).  1 for amax == 0; never
// below 2^-126, so s is a normal float (an amax under 2^-118 then gives amax / s < 256).
__device__ __forceinline__ float fp8_block_scale(float amax) {
  if (amax == 0.f) return 1.0f;
  const uint32_t b = __float_as_uint(amax);
  const int e = (int)(b >> 23) - 8 + ((b & 0x7fffffu) > 0x600000u ? 1 : 0);
  return __uint_as_float((uint32_t)(e < 1 ? 1 : e) << 23);
}
// two fp32 values -> e4m3 (round to nearest even, saturating), lo in the low byte
__device__ __forceinline__ uint16_t cvt_e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// named barrier for a subset of warps (id 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// arrive without waiting (the producer side of a named-barrier hand-off)
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace esmb200
