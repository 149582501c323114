// esm_b200 — embedding-based pairwise alignment (esm_b200/align.py), the definition in include/esmb200.h at
// esmb200_align_similarity / esmb200_align.
//
// P pairs, pair p a query of La rows and a target of Lb rows (fp16, normalised, D columns). Offsets are int64 device
// arrays: query rows [q_off[p], q_off[p+1]), target rows [t_off[p], t_off[p+1]), S' at s_off[p] as [La, Lb] fp32.
//   align_sim_kernel     grid (P, splits): a CTA walks its pair's 64 x 64 tiles of S = A B^T with stride `splits`,
//                        mma.sync m16n8k16 (fp16 operands, fp32 accumulation), K in 64-wide slabs through shared
//                        memory; rows past La / Lb are zero-filled and never stored.
//   align_stats_kernel   grid (P, splits): mean and population standard deviation of every row (one warp, lanes
//                        strided, xor butterfly) and every column (one thread, rows in order) of S, two passes in
//                        fp64; each statistic is reduced by one warp or thread in a fixed order, so S' is
//                        bit-reproducible without atomics. (mu, sd) fp32 pairs go to scratch.
//   align_zscore_kernel  grid (P, splits): S'[i,j] = 0.5 * ((S - mu_r) / sd_r + (S - mu_c) / sd_c), a term 0 where
//                        its sd is 0, in place.
//   align_dp_kernel      one warp per pair. Lane t owns query row i = 32 b + t + 1 of row block b and runs a wavefront
//                        across target columns 0 ... Lb: at step s lane t computes column j = s - t, taking H and F of
//                        row i - 1 from lane t - 1 by shuffle (lane 0 from the previous block's bottom row in the
//                        border buffer, or from row 0 itself for block 0). One direction byte per cell; the 32 bytes
//                        of one step are contiguous (the diagonal layout below), so each step is one 32-byte store.
//   align_trace_kernel   one thread per pair: the traceback state machine over the direction bytes, ops reversed
//                        into query->target order in place.
// Every candidate costs one fp32 add or subtract (__fadd_rn / __fsub_rn: nothing is contracted), so a float32 numpy
// restatement gives the same bits.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace esmb200 {

constexpr int kAlignTile = 64;      // S tile edge and K slab of align_sim_kernel
constexpr int kAlignSimThreads = 128;
constexpr int kAlignStatThreads = 256;
constexpr int kAlignSmemPitch = 72;  // fp16 per staged row: 64 + 8, so the fragment loads hit distinct banks

// direction byte: bits 0-1 the source of H (0 zero, 1 diagonal, 2 E, 3 F), bit 2 E extended, bit 3 F extended
constexpr uint8_t kDirZero = 0, kDirDiag = 1, kDirE = 2, kDirF = 3, kDirEExt = 4, kDirFExt = 8;

// Scratch of P pairs with n_q query rows, n_t target rows and n_cells cells in all (esmb200_align_scratch_bytes):
//   direction bytes  pair p at align32(s_off[p] + 32 (q_off[p] + t_off[p]) + 1024 p): ceil(La / 32) row blocks of
//                    (Lb + 32) steps x 32 lanes, cell (i, j) (1-based) at ((i-1)/32 * (Lb + 32) + j + (i-1)%32) * 32
//                    + (i-1)%32; at most La Lb + 32 La + 31 Lb + 992 bytes, so pair p + 1's region starts past it
//   border rows      pair p at float2 offset 2 (t_off[p] + p): two buffers of Lb + 1 (H, F) pairs
//   statistics       (mu, sd) float2 per query row at q_off[p] + i and per target column at n_q + t_off[p] + j (the
//                    z-score of esmb200_align_similarity; the same scratch serves both calls)
struct AlignScratch {
  size_t dir_bytes, border_off, stats_off, bytes;
};

inline AlignScratch align_scratch(int64_t P, int64_t n_q, int64_t n_t, int64_t n_cells) {
  AlignScratch s;
  s.dir_bytes = (size_t)(n_cells + 32 * (n_q + n_t) + 1024 * P + 32);
  s.border_off = (s.dir_bytes + 255) / 256 * 256;
  s.stats_off = s.border_off + (size_t)(16 * (n_t + P) + 255) / 256 * 256;
  s.bytes = s.stats_off + (size_t)(8 * (n_q + n_t));
  return s;
}

struct AlignPair {
  int64_t q0, t0, s0;
  int La, Lb;
};

__device__ __forceinline__ bool align_pair(const int64_t* q_off, const int64_t* t_off, const int64_t* s_off, int p,
                                           AlignPair& a) {
  a.q0 = q_off[p];
  a.t0 = t_off[p];
  a.s0 = s_off[p];
  const int64_t La = q_off[p + 1] - a.q0, Lb = t_off[p + 1] - a.t0;
  a.La = (int)La;
  a.Lb = (int)Lb;
  return La >= 1 && Lb >= 1 && La <= INT32_MAX && Lb <= INT32_MAX;
}

// ---- similarity -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAlignSimThreads)
align_sim_kernel(const __half* __restrict__ q, const __half* __restrict__ t, int D, const int64_t* q_off,
                 const int64_t* t_off, const int64_t* s_off, float* __restrict__ out) {
  __shared__ __align__(16) __half sa[kAlignTile * kAlignSmemPitch];
  __shared__ __align__(16) __half sb[kAlignTile * kAlignSmemPitch];
  AlignPair a;
  if (!align_pair(q_off, t_off, s_off, blockIdx.x, a)) return;
  const int tiles_m = (a.La + kAlignTile - 1) / kAlignTile, tiles_n = (a.Lb + kAlignTile - 1) / kAlignTile;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;  // this warp's 32 x 32 quarter of the tile
  for (int64_t tile = blockIdx.y; tile < (int64_t)tiles_m * tiles_n; tile += gridDim.y) {
    const int m0 = (int)(tile / tiles_n) * kAlignTile, n0 = (int)(tile % tiles_n) * kAlignTile;
    float acc[2][4][4] = {};
    for (int k0 = 0; k0 < D; k0 += kAlignTile) {
      __syncthreads();
      for (int v = tid; v < kAlignTile * 8; v += kAlignSimThreads) {  // 64 rows x 8 16-byte vectors per operand
        const int r = v >> 3, col = (v & 7) * 8;
        uint4 xa = make_uint4(0, 0, 0, 0), xb = make_uint4(0, 0, 0, 0);
        if (m0 + r < a.La) xa = *reinterpret_cast<const uint4*>(q + (a.q0 + m0 + r) * D + k0 + col);
        if (n0 + r < a.Lb) xb = *reinterpret_cast<const uint4*>(t + (a.t0 + n0 + r) * D + k0 + col);
        *reinterpret_cast<uint4*>(sa + r * kAlignSmemPitch + col) = xa;
        *reinterpret_cast<uint4*>(sb + r * kAlignSmemPitch + col) = xb;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < kAlignTile; kk += 16) {
        uint32_t fa[2][4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          const __half* base = sa + (wm + mi * 16 + g) * kAlignSmemPitch + kk + 2 * c;
          fa[mi][0] = *reinterpret_cast<const uint32_t*>(base);
          fa[mi][1] = *reinterpret_cast<const uint32_t*>(base + 8 * kAlignSmemPitch);
          fa[mi][2] = *reinterpret_cast<const uint32_t*>(base + 8);
          fa[mi][3] = *reinterpret_cast<const uint32_t*>(base + 8 * kAlignSmemPitch + 8);
        }
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          const __half* base = sb + (wn + ni * 8 + g) * kAlignSmemPitch + kk + 2 * c;
          const uint32_t b0 = *reinterpret_cast<const uint32_t*>(base);
          const uint32_t b1 = *reinterpret_cast<const uint32_t*>(base + 8);
#pragma unroll
          for (int mi = 0; mi < 2; ++mi) mma16816(acc[mi][ni], fa[mi], b0, b1);
        }
      }
    }
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = m0 + wm + mi * 16 + g + 8 * h, j = n0 + wn + ni * 8 + 2 * c;
          if (i >= a.La) continue;
          float* row = out + a.s0 + (int64_t)i * a.Lb;
          if (j < a.Lb) row[j] = acc[mi][ni][2 * h];
          if (j + 1 < a.Lb) row[j + 1] = acc[mi][ni][2 * h + 1];
        }
  }
}

__global__ void __launch_bounds__(kAlignStatThreads)
align_stats_kernel(const float* __restrict__ s, const int64_t* q_off, const int64_t* t_off, const int64_t* s_off,
                   int64_t n_q, float2* __restrict__ stats) {
  AlignPair a;
  if (!align_pair(q_off, t_off, s_off, blockIdx.x, a)) return;
  const float* S = s + a.s0;
  const int warps = kAlignStatThreads / 32, lane = threadIdx.x & 31;
  for (int i = blockIdx.y * warps + (threadIdx.x >> 5); i < a.La; i += gridDim.y * warps) {
    const float* row = S + (int64_t)i * a.Lb;
    double sum = 0.0;
    for (int j = lane; j < a.Lb; j += 32) sum += row[j];
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const double mu = sum / a.Lb;
    double ss = 0.0;
    for (int j = lane; j < a.Lb; j += 32) ss += (row[j] - mu) * (row[j] - mu);
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if (lane == 0) stats[a.q0 + i] = make_float2((float)mu, (float)sqrt(ss / a.Lb));
  }
  for (int j = blockIdx.y * kAlignStatThreads + threadIdx.x; j < a.Lb; j += gridDim.y * kAlignStatThreads) {
    double sum = 0.0;
    for (int i = 0; i < a.La; ++i) sum += S[(int64_t)i * a.Lb + j];
    const double mu = sum / a.La;
    double ss = 0.0;
    for (int i = 0; i < a.La; ++i) {
      const double d = S[(int64_t)i * a.Lb + j] - mu;
      ss += d * d;
    }
    stats[n_q + a.t0 + j] = make_float2((float)mu, (float)sqrt(ss / a.La));
  }
}

__global__ void __launch_bounds__(kAlignStatThreads)
align_zscore_kernel(float* __restrict__ s, const int64_t* q_off, const int64_t* t_off, const int64_t* s_off,
                    int64_t n_q, const float2* __restrict__ stats) {
  AlignPair a;
  if (!align_pair(q_off, t_off, s_off, blockIdx.x, a)) return;
  const int64_t cells = (int64_t)a.La * a.Lb;
  for (int64_t x = (int64_t)blockIdx.y * kAlignStatThreads + threadIdx.x; x < cells;
       x += (int64_t)gridDim.y * kAlignStatThreads) {
    const int i = (int)(x / a.Lb), j = (int)(x % a.Lb);
    const float v = s[a.s0 + x];
    const float2 r = stats[a.q0 + i], col = stats[n_q + a.t0 + j];
    const float tr = r.y > 0.f ? __fdiv_rn(__fsub_rn(v, r.x), r.y) : 0.f;
    const float tc = col.y > 0.f ? __fdiv_rn(__fsub_rn(v, col.x), col.y) : 0.f;
    s[a.s0 + x] = __fmul_rn(0.5f, __fadd_rn(tr, tc));
  }
}

// ---- dynamic programme --------------------------------------------------------------------------------------------
struct AlignBest {
  float h;
  int i, j;
};

__device__ __forceinline__ bool align_better(const AlignBest& x, const AlignBest& y) {  // x before y
  return x.h > y.h || (x.h == y.h && (x.i < y.i || (x.i == y.i && x.j < y.j)));
}

__global__ void __launch_bounds__(32)
align_dp_kernel(const float* __restrict__ s, const int64_t* q_off, const int64_t* t_off, const int64_t* s_off,
                int local, float o, float e, uint8_t* __restrict__ scratch, size_t border_off, float* scores,
                int32_t* spans) {
  const int p = blockIdx.x, t = threadIdx.x;
  AlignPair a;
  if (!align_pair(q_off, t_off, s_off, p, a)) {
    if (t == 0) {
      scores[p] = __int_as_float(0x7fc00000);
      for (int k = 0; k < 4; ++k) spans[4 * p + k] = -1;
    }
    return;
  }
  const float NEG = -INFINITY;
  const float* S = s + a.s0;
  uint8_t* dir = scratch + ((a.s0 + 32 * (a.q0 + a.t0) + 1024 * (int64_t)p + 31) & ~(int64_t)31);
  float2* border = reinterpret_cast<float2*>(scratch + border_off) + 2 * (a.t0 + p);  // 2 x (Lb + 1) (H, F)
  const int blocks = (a.La + 31) / 32, steps = a.Lb + 32;
  AlignBest best = {0.f, 0, 0};  // local: row 0 and column 0 hold H = 0, so (0, 0) wins a score of 0
  float final_h = 0.f;
  for (int b = 0; b < blocks; ++b) {
    const int i = 32 * b + t + 1;
    const bool row_ok = i <= a.La;
    const float2* up_buf = border + (b & 1) * (a.Lb + 1);
    float2* down_buf = border + ((b + 1) & 1) * (a.Lb + 1);
    const bool write_down = t == 31 && b + 1 < blocks;
    float h_left = 0.f, e_left = NEG, h_diag = 0.f;  // H[i][j-1], E[i][j-1], H[i-1][j-1]
    float h_out = 0.f, f_out = NEG;                  // this lane's H[i][j], F[i][j] of the last step
    float h0 = 0.f, e0 = NEG;                        // row 0 (block 0, lane 0): H[0][j], E[0][j]
    const float* srow = S + (int64_t)(i - 1) * a.Lb;
    uint8_t* dstep = dir + (int64_t)b * steps * 32 + t;
    for (int st = 0; st < steps; ++st) {
      float up_h = __shfl_up_sync(0xffffffffu, h_out, 1), up_f = __shfl_up_sync(0xffffffffu, f_out, 1);
      const int j = st - t;
      if (j < 0 || j > a.Lb || !row_ok) continue;
      if (t == 0) {
        if (b == 0) {  // row 0 itself
          if (j > 0 && !local) {
            const float op = __fsub_rn(h0, o), ex = __fsub_rn(e0, e);
            e0 = ex > op ? ex : op;
            h0 = e0;
          }
          up_h = h0;
          up_f = NEG;
        } else {
          const float2 v = up_buf[j];
          up_h = v.x;
          up_f = v.y;
        }
      }
      const float fo = __fsub_rn(up_h, o), fx = __fsub_rn(up_f, e);
      const float f = fx > fo ? fx : fo;
      float h;
      if (j == 0) {  // column 0: H = 0 (local) or F (global), E = -inf; no direction byte
        h = local ? 0.f : f;
        e_left = NEG;
        h_out = h;
        f_out = local ? NEG : f;
      } else {
        const float eo = __fsub_rn(h_left, o), ex = __fsub_rn(e_left, e);
        const float ev = ex > eo ? ex : eo;
        const float dg = __fadd_rn(h_diag, __ldg(srow + j - 1));
        h = dg;
        uint8_t src = kDirDiag;
        if (ev > h) { h = ev; src = kDirE; }
        if (f > h) { h = f; src = kDirF; }
        if (local && 0.f > h) { h = 0.f; src = kDirZero; }
        dstep[(int64_t)st * 32] = (uint8_t)(src | (ex > eo ? kDirEExt : 0) | (fx > fo ? kDirFExt : 0));
        e_left = ev;
        h_out = h;
        f_out = f;
        if (local && h > best.h) best = {h, i, j};  // this lane's row in increasing j: strict > keeps the first
        if (!local && i == a.La && j == a.Lb) final_h = h;
      }
      h_left = h;
      h_diag = up_h;
      if (write_down) down_buf[j] = make_float2(h_out, f_out);
    }
    __syncwarp();
  }
  if (local) {
    for (int off = 16; off > 0; off >>= 1) {
      AlignBest other = {__shfl_xor_sync(0xffffffffu, best.h, off), __shfl_xor_sync(0xffffffffu, best.i, off),
                         __shfl_xor_sync(0xffffffffu, best.j, off)};
      if (align_better(other, best)) best = other;
    }
    if (t == 0) {
      scores[p] = best.h;
      spans[4 * p + 1] = best.i;
      spans[4 * p + 3] = best.j;
    }
  } else if (t == (a.La - 1) % 32) {
    scores[p] = final_h;
    spans[4 * p + 1] = a.La;
    spans[4 * p + 3] = a.Lb;
  }
}

__global__ void __launch_bounds__(128)
align_trace_kernel(const int64_t* q_off, const int64_t* t_off, const int64_t* s_off, int P, int local,
                   const uint8_t* __restrict__ scratch, int32_t* spans, uint8_t* ops, int32_t* n_ops) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  AlignPair a;
  if (!align_pair(q_off, t_off, s_off, p, a)) {
    n_ops[p] = -1;
    return;
  }
  const uint8_t* dir = scratch + ((a.s0 + 32 * (a.q0 + a.t0) + 1024 * (int64_t)p + 31) & ~(int64_t)31);
  uint8_t* out = ops + a.q0 + a.t0;  // La + Lb bytes per pair
  int i = spans[4 * p + 1], j = spans[4 * p + 3], n = 0, state = 0;  // state 0 H, 1 E, 2 F
  for (;;) {
    if (i == 0 || j == 0) {
      if (local || (i == 0 && j == 0)) break;
      out[n++] = i == 0 ? 'T' : 'Q';  // global: the border runs straight to (0, 0)
      if (i == 0) --j; else --i;
      continue;
    }
    const int r = i - 1;
    const uint8_t d = dir[((int64_t)(r >> 5) * (a.Lb + 32) + j + (r & 31)) * 32 + (r & 31)];
    if (state == 0) {
      const int src = d & 3;
      if (src == kDirZero) break;
      if (src == kDirDiag) { out[n++] = 'M'; --i; --j; }
      else state = src == kDirE ? 1 : 2;
    } else if (state == 1) {
      out[n++] = 'T';
      --j;
      state = (d & kDirEExt) ? 1 : 0;
    } else {
      out[n++] = 'Q';
      --i;
      state = (d & kDirFExt) ? 2 : 0;
    }
  }
  for (int k = 0; k < n / 2; ++k) {
    const uint8_t x = out[k];
    out[k] = out[n - 1 - k];
    out[n - 1 - k] = x;
  }
  spans[4 * p] = i;
  spans[4 * p + 2] = j;
  n_ops[p] = n;
}

}  // namespace esmb200
