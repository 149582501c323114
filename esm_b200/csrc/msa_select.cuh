// esm_b200 — greedy maximum / minimum-Hamming row selection of a deep alignment for the MSA Transformer
// (esm_b200/msa_select.py), the definition in include/esmb200.h at esmb200_msa_greedy_select.
//
// One alignment rows uint8 [N, ld] (ld a multiple of 16, the padding bytes equal in every row). Step t = 1 ... k - 1:
//   msa_select_step_kernel  one launch per step, one block per 256 rows, nothing read back by the host:
//     1. the Hamming count of every row against the row picked at step t - 1 (selected[t - 1], read on the device), the
//        picked row staged in shared memory, 8 lanes per row with 16-byte loads -> counts[t - 1, :] (uint16)
//     2. per unpicked candidate j the score numpy's mean(0) gives (pairwise sum of d_1[j] ... d_t[j], d = count / C,
//        then / t), in fp64 with __dadd_rn / __ddiv_rn so nothing is contracted or reassociated
//     3. (score, index) reduced to the best with the smallest index on ties, per block and then by the last block to
//        finish (an atomic ticket): max / min with that tie rule is order-independent, so the winner is deterministic.
//        The last block writes selected[t], marks the row picked and resets the ticket.
// msa_select_init_kernel runs once before step 1: selected[0] = 0, only row 0 picked, the table d[c] = c / C.
#pragma once

#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

namespace esmb200 {

constexpr int kSelThreads = 256;  // rows per block of the step kernel
constexpr int kSelLanes = 8;      // lanes per row when counting
constexpr int kSelDepth = 26;     // pairwise-sum split levels: a node of n > 128 terms has children of at most
                                  // n / 2 + 8, so 25 levels take any n < 2^31 to a leaf of at most 128

// Scratch layout (each array 256-byte aligned): counts uint16 [k - 1, N] | d fp64 [C + 1] | picked uint8 [N] |
// block partials (fp64 score [blocks], int32 index [blocks]) | ticket uint32.
struct MsaSelectScratch {
  uint16_t* counts;
  double* dist;
  uint8_t* picked;
  double* part_score;
  int* part_index;
  unsigned* ticket;
  size_t bytes;
};

inline size_t sel_align(size_t v) { return (v + 255) / 256 * 256; }

inline MsaSelectScratch msa_select_scratch(char* base, int N, int C, int k) {
  const size_t n = (size_t)N, blocks = (n + kSelThreads - 1) / kSelThreads;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off = sel_align(off + bytes);
    return p;
  };
  MsaSelectScratch s;
  s.counts = reinterpret_cast<uint16_t*>(take((size_t)(k > 1 ? k - 1 : 0) * n * 2));
  s.dist = reinterpret_cast<double*>(take(((size_t)C + 1) * 8));
  s.picked = reinterpret_cast<uint8_t*>(take(n));
  s.part_score = reinterpret_cast<double*>(take(blocks * 8));
  s.part_index = reinterpret_cast<int*>(take(blocks * 4));
  s.ticket = reinterpret_cast<unsigned*>(take(4));
  s.bytes = off;
  return s;
}

__global__ void __launch_bounds__(256)
msa_select_init_kernel(int N, int C, double* __restrict__ dist, uint8_t* __restrict__ picked,
                       unsigned* __restrict__ ticket, int64_t* __restrict__ selected) {
  const int n = N > C + 1 ? N : C + 1;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
    if (i < N) picked[i] = i == 0;
    if (i <= C) dist[i] = __ddiv_rn((double)i, (double)C);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    selected[0] = 0;
    *ticket = 0u;
  }
}

// numpy's pairwise_sum (numpy/_core/src/umath/loops_utils.h.src) of the terms d[counts[(lo + i) * N]], i < n <= 128:
// below 8 terms a sequential sum from +0; otherwise eight strided accumulators over the first n - n % 8 terms, combined
// as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the tail added in order.
__device__ __forceinline__ double sel_leaf(const uint16_t* __restrict__ c, int64_t N, int lo, int n,
                                           const double* __restrict__ dist) {
  const uint16_t* p = c + (int64_t)lo * N;
  if (n < 8) {
    double res = 0.0;
    for (int i = 0; i < n; ++i) res = __dadd_rn(res, dist[p[(int64_t)i * N]]);
    return res;
  }
  double r[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) r[u] = dist[p[(int64_t)u * N]];
  int i = 8;
  for (; i < n - n % 8; i += 8) {
#pragma unroll
    for (int u = 0; u < 8; ++u) r[u] = __dadd_rn(r[u], dist[p[(int64_t)(i + u) * N]]);
  }
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __dadd_rn(res, dist[p[(int64_t)i * N]]);
  return res;
}

// Above 128 terms numpy splits at n2 = n / 2 - (n / 2) % 8 and adds the two halves' sums. The tree depends only on n,
// so every thread walks the same one: an iterative post-order with a per-thread stack of waiting nodes (the right
// child's range, and its left sum once known), kSelDepth deep, in place of recursion.
__device__ __forceinline__ double sel_pairwise(const uint16_t* __restrict__ c, int64_t N, int n,
                                               const double* __restrict__ dist) {
  int st_lo[kSelDepth], st_n[kSelDepth];
  double st_left[kSelDepth];
  bool st_has_left[kSelDepth];
  int sp = 0, lo = 0;
  while (true) {
    while (n > 128) {
      int n2 = n / 2;
      n2 -= n2 % 8;
      st_lo[sp] = lo + n2;
      st_n[sp] = n - n2;
      st_has_left[sp] = false;
      ++sp;
      n = n2;
    }
    double v = sel_leaf(c, N, lo, n, dist);
    while (sp > 0 && st_has_left[sp - 1]) {
      v = __dadd_rn(st_left[sp - 1], v);
      --sp;
    }
    if (sp == 0) return v;
    st_left[sp - 1] = v;
    st_has_left[sp - 1] = true;
    lo = st_lo[sp - 1];
    n = st_n[sp - 1];
  }
}

template <bool kMax>
__device__ __forceinline__ bool sel_better(double s, int i, double bs, int bi) {
  return (kMax ? s > bs : s < bs) || (s == bs && i < bi);
}

// Block-wide (score, index) reduction; the result is returned to every thread.
template <bool kMax>
__device__ __forceinline__ void sel_block_best(double& s, int& i, double* red_s, int* red_i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
    if (sel_better<kMax>(s2, i2, s, i)) {
      s = s2;
      i = i2;
    }
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    red_s[warp] = s;
    red_i[warp] = i;
  }
  __syncthreads();
  s = red_s[0];
  i = red_i[0];
#pragma unroll
  for (int w = 1; w < kSelThreads / 32; ++w)
    if (sel_better<kMax>(red_s[w], red_i[w], s, i)) {
      s = red_s[w];
      i = red_i[w];
    }
  __syncthreads();
}

// Step t >= 1. Dynamic shared memory: ld bytes (the picked row).
template <bool kMax>
__global__ void __launch_bounds__(kSelThreads)
msa_select_step_kernel(const uint8_t* __restrict__ rows, int64_t ld, int N, int t, int64_t* __restrict__ selected,
                       MsaSelectScratch s) {
  extern __shared__ uint4 s_pick[];
  __shared__ double red_s[kSelThreads / 32];
  __shared__ int red_i[kSelThreads / 32];
  __shared__ bool is_last;
  const int nv = (int)(ld / 16);
  const uint4* pick = reinterpret_cast<const uint4*>(rows + selected[t - 1] * ld);
  for (int v = threadIdx.x; v < nv; v += kSelThreads) s_pick[v] = pick[v];
  __syncthreads();

  // 1. counts[t - 1, j] for this block's rows: group g of 8 lanes takes rows j0 + g + 32 m.
  const int64_t j0 = (int64_t)blockIdx.x * kSelThreads;
  const int g = threadIdx.x / kSelLanes, lane = threadIdx.x % kSelLanes;
  uint16_t* crow = s.counts + (int64_t)(t - 1) * N;
  for (int m = 0; m < kSelThreads / 32; ++m) {
    const int64_t j = j0 + g + 32 * m;
    unsigned bits = 0;
    if (j < N) {
      const uint4* row = reinterpret_cast<const uint4*>(rows + (int64_t)j * ld);
      for (int v = lane; v < nv; v += kSelLanes) {
        const uint4 a = row[v], b = s_pick[v];
        bits += __popc(__vcmpne4(a.x, b.x)) + __popc(__vcmpne4(a.y, b.y)) + __popc(__vcmpne4(a.z, b.z)) +
                __popc(__vcmpne4(a.w, b.w));
      }
    }
#pragma unroll
    for (int o = kSelLanes / 2; o > 0; o >>= 1) bits += __shfl_xor_sync(0xffffffffu, bits, o);
    if (lane == 0 && j < N) crow[j] = (uint16_t)(bits >> 3);  // __vcmpne4 sets 8 bits per differing byte
  }
  __syncthreads();

  // 2. the candidate's score.
  const int64_t j = j0 + threadIdx.x;
  double best = kMax ? -INFINITY : INFINITY;
  int bi = INT_MAX;
  if (j < N && !s.picked[j]) {
    best = __ddiv_rn(sel_pairwise(s.counts + j, N, t, s.dist), (double)t);
    bi = (int)j;
  }

  // 3. the block's best, then the grid's in the last block to finish.
  sel_block_best<kMax>(best, bi, red_s, red_i);
  if (threadIdx.x == 0) {
    s.part_score[blockIdx.x] = best;
    s.part_index[blockIdx.x] = bi;
    __threadfence();
    is_last = atomicAdd(s.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  best = kMax ? -INFINITY : INFINITY;
  bi = INT_MAX;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += kSelThreads) {
    const double s2 = __ldcg(s.part_score + b);
    const int i2 = __ldcg(s.part_index + b);
    if (sel_better<kMax>(s2, i2, best, bi)) {
      best = s2;
      bi = i2;
    }
  }
  sel_block_best<kMax>(best, bi, red_s, red_i);
  if (threadIdx.x == 0) {
    selected[t] = bi;
    s.picked[bi] = 1;
    *s.ticket = 0u;
  }
}

}  // namespace esmb200
