// esm_b200 — exact k-nearest-neighbour search over embeddings (esm_b200/search.py): a wgmma similarity GEMM whose
// epilogue keeps each query's top k, so the [Q, N] score matrix never reaches HBM.  Definition in include/esmb200.h at
// esmb200_knn_search.
//
//   s(i, j) = alpha * (A_i . X_j) + beta_j   (fp16 operands, fp32 accumulation), j in [0, N), j != i + self_offset
//
// Ranking key.  A candidate is the 64-bit key (ord(s) << 32) | (2^32 - 1 - j), ord the order-preserving map of fp32
// bits to uint32.  Keys are distinct for distinct j and order candidates by (score descending, index ascending), so the
// top k of a set of keys is one well-defined set whatever order the candidates arrive in.  Key 0 is below every finite
// score and marks an empty slot.
//
// knn_topk_kernel: one CTA per (64-query block, database stripe); blockIdx.x = stripe * query_blocks + block, so the
// CTAs resident at one time share a stripe and read its tiles from the L2.
//   * warpgroup 0: one thread streams 64-wide K slabs of the query block (64 rows, 8 KB) and of a 256-row database
//     tile (32 KB) through a 3-stage TMA ring (128B swizzle); TMA zero-fills rows >= Q and >= N;
//   * warpgroup 1: wgmma m64n256k16 into 128 fp32 accumulators per thread, then the epilogue: s = alpha acc + beta_j
//     in registers, key > the row's k-th best key (a warpgroup-wide OR first, so a tile without a survivor costs one
//     barrier); survivors go to the row's 64-entry queue in shared memory, 32 columns at a time; when a row's queue
//     could overflow with the next 32, every row's queue is sorted (warp bitonic sort) and merged into its k-list by
//     rank.  Rows >= Q, columns >= N and j == i + self_offset never produce a candidate.  The threshold only rises,
//     and queued candidates are never lost, so the list is the exact top k of the stripe.
//   * the k-list of each valid row is written to scratch keys[stripe, q, 0..k) (descending, 0 past the stripe's
//     candidates).
// knn_merge_kernel: one block per query merges the S stripe lists (k rounds of a block-wide maximum over the list
// heads) and decodes the keys to fp32 scores and int64 indices.
//
// Streamed search (esmb200_knn_search_accumulate): the database arrives in chunks; a chunk of n rows holds global rows
// [row0, row0 + n), and candidate keys carry the global index, so a key means the same thing in every chunk.  A running
// list keys [Q, k] (0 = empty slot) holds the top k of the chunks seen so far.  knn_topk_kernel seeds each row's
// threshold with the running k-th key: a candidate at or below it cannot enter the final top k, so seeding changes no
// result, and once the list has filled most tiles end at the warpgroup OR.  knn_merge_kernel<ACC> then merges the
// stripe lists and the running list (copied to shared memory first, since it is overwritten in place) and writes keys
// back undecoded; knn_decode_kernel decodes the final list once.
//
// Shared memory of knn_topk_kernel (k <= 128): ring 3 x (8 + 32) KB = 120 KB, k-lists 64 x 128 x 8 B = 64 KB, queues
// 64 x 64 x 8 B = 32 KB, thresholds 512 B, queue counts 256 B, barriers, 1 KB alignment slack: 223,232 B of 232,448.
// 64 query rows per CTA: 128 rows would need 128 KB of k-lists at k = 128, leaving no room for a 3-stage ring.
#pragma once

#include "common.cuh"

namespace esmb200 {

namespace knn_cfg {
constexpr int BLOCK_M = 64;    // query rows per CTA
constexpr int BLOCK_N = 256;   // database rows per tile
constexpr int BLOCK_K = 64;
constexpr int STAGES = 3;
constexpr int MAX_K = 128;
constexpr int QCAP = 64;       // queue entries per row
constexpr int CHUNK = 32;      // columns pushed between overflow checks
constexpr int MAX_SPLITS = 1024;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 8 KB
constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;  // 32 KB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int LIST_BYTES = BLOCK_M * MAX_K * 8;
constexpr int QUEUE_BYTES = BLOCK_M * QCAP * 8;
constexpr int NUM_THREADS = 256;  // warpgroup 0: TMA producer, warpgroup 1: MMA + top-k epilogue
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + LIST_BYTES + QUEUE_BYTES + BLOCK_M * 8 + BLOCK_M * 4 + 256 + 1024;
static_assert(SMEM_BYTES <= 232448, "knn_topk_kernel shared memory");
}  // namespace knn_cfg

// A list-scan work item: query rows [g0, g1) (at most BLOCK_M, all probing one list) against stored rows [r0, r1) (a
// stripe of that list, tiles starting at r0); the rows' partial lists go to keys[pbase[g] + stripe].
struct IvfItem {
  int32_t g0, g1, r0, r1, stripe;
};

struct KnnParams {
  int Q, D, k;
  int64_t N;
  int tiles_per_stripe;  // 256-row tiles per stripe
  int query_blocks;
  const float* beta;     // [N] or nullptr
  float alpha;
  int64_t self_offset;   // < 0: none; in global rows
  int64_t row0;          // global index of the chunk's row 0 (0 for esmb200_knn_search)
  union {  // one mode's pointers: the range fields overlay the top-k ones, so the parameter block keeps its size
    struct {
      const unsigned long long* seed;  // running list [Q, k] whose k-th key seeds the thresholds, or nullptr
      unsigned long long* keys;  // scratch [splits, Q, k]; list scan: [Q, R, k] (the query's partial lists, ragged)
      // list scan (LISTS) only
      const IvfItem* items;  // one work item per CTA
      const int64_t* ids;           // [N] original row of each stored row: the key's index
      const int64_t* gself;         // [query rows] the original row each query row leaves out (< 0: none), or nullptr
      const int* pbase;             // [query rows] partial-list index of the row's stripe 0 (< 0: the row writes nothing)
    };
    struct {  // range search (RANGE) only
      const float* tau;                  // [Q] each query's threshold: its hits are the candidates with s >= tau
      unsigned long long* hit_keys;      // [hit_cap] appended hit keys
      int* hit_rows;                     // [hit_cap] the query row of each appended hit
      unsigned long long* hit_counts;    // [Q] hits per query, counted past hit_cap
      unsigned long long* hit_total;     // hits appended in all, counted past hit_cap
      int64_t hit_cap;
    };
  };
};

__device__ __forceinline__ unsigned long long knn_key(float s, int64_t j) {
  const uint32_t u = __float_as_uint(s);
  const uint32_t o = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)o << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)j);
}

// the inverse of knn_key: the fp32 score and the index
__device__ __forceinline__ void knn_decode_key(unsigned long long key, float* score, int64_t* idx) {
  const uint32_t o = (uint32_t)(key >> 32);
  const uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
  *score = __uint_as_float(u);
  *idx = (int64_t)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull));
}

// warpgroup-wide OR (bar.red on a named barrier: also a barrier with bar.sync's memory ordering)
__device__ __forceinline__ bool knn_bar_or(uint32_t id, bool v) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "bar.red.or.pred q, %2, 128, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}"
      : "=r"(r)
      : "r"((uint32_t)v), "r"(id)
      : "memory");
  return r != 0;
}

// Merge one row's queue (cnt > 0 entries) into its k-list; one warp, called with a warp-uniform row.  SEEDED: the
// threshold may start above the list's k-th key (streamed search), so a merge keeps the larger of the two.
template <bool SEEDED>
__device__ __forceinline__ void knn_merge_row(unsigned long long* list, unsigned long long* queue, int* cnt,
                                              unsigned long long* th, int k, uint32_t lane) {
  const int n = *cnt < knn_cfg::QCAP ? *cnt : knn_cfg::QCAP;
  unsigned long long v[2];
#pragma unroll
  for (int sl = 0; sl < 2; ++sl) v[sl] = (int)(32 * sl + lane) < n ? queue[32 * sl + lane] : 0ull;
  // bitonic sort of the 64 keys, descending; element x = 32 slot + lane
#pragma unroll
  for (int size = 2; size <= 64; size <<= 1) {
#pragma unroll
    for (int d = size / 2; d > 0; d >>= 1) {
      if (d == 32) {  // size == 64: the two slots of one lane
        const unsigned long long hi = v[0] > v[1] ? v[0] : v[1], lo = v[0] > v[1] ? v[1] : v[0];
        v[0] = hi;
        v[1] = lo;
      } else {
#pragma unroll
        for (int sl = 0; sl < 2; ++sl) {
          const uint32_t x = 32 * sl + lane;
          const unsigned long long p = __shfl_xor_sync(0xffffffffu, v[sl], d);
          const bool want_max = ((x & d) == 0) == ((x & size) == 0);
          v[sl] = want_max ? (v[sl] > p ? v[sl] : p) : (v[sl] < p ? v[sl] : p);
        }
      }
    }
  }
#pragma unroll
  for (int sl = 0; sl < 2; ++sl) queue[32 * sl + lane] = v[sl];
  __syncwarp();
  // merge by rank: a list entry goes to i + #(queue > it), a queue entry to j + #(list >= it); ranks < k are kept
  unsigned long long lv[knn_cfg::MAX_K / 32];
  int lr[knn_cfg::MAX_K / 32], qr[2];
#pragma unroll
  for (int t = 0; t < knn_cfg::MAX_K / 32; ++t) {
    const int i = 32 * t + (int)lane;
    lr[t] = knn_cfg::MAX_K;
    if (i < k) {
      const unsigned long long x = list[i];
      int lo = 0, hi = knn_cfg::QCAP;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (queue[mid] > x) lo = mid + 1; else hi = mid;
      }
      lv[t] = x;
      lr[t] = i + lo;
    }
  }
#pragma unroll
  for (int sl = 0; sl < 2; ++sl) {
    int lo = 0, hi = k;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (list[mid] >= v[sl]) lo = mid + 1; else hi = mid;
    }
    qr[sl] = 32 * sl + (int)lane + lo;
  }
  __syncwarp();
#pragma unroll
  for (int t = 0; t < knn_cfg::MAX_K / 32; ++t)
    if (lr[t] < k) list[lr[t]] = lv[t];
#pragma unroll
  for (int sl = 0; sl < 2; ++sl)
    if (qr[sl] < k) list[qr[sl]] = v[sl];
  __syncwarp();
  if (lane == 0) {
    *th = (SEEDED && *th > list[k - 1]) ? *th : list[k - 1];
    *cnt = 0;
  }
  __syncwarp();
}

// STREAM: a chunk of a streamed search (row0 and the seeded thresholds); without it the kernel is the resident one,
// with no code for either.  LISTS: the inverted-file list scan (esmb200_ivf_search): CTA b runs work item items[b],
// columns outside [r0, r1) and query rows outside [g0, g1) produce no candidate, a key's index is ids[j] and a row
// leaves out the column whose id is gself[row]; without it none of this is compiled.  RANGE: the range search
// (esmb200_knn_range): global indices from row0, each row's threshold fixed at (ord(tau) << 32) - 1, so key > th
// exactly when s >= tau, and a queue that could overflow is flushed to the global hit buffer instead of merged into a
// k-list; no k-list is kept or written.
template <bool STREAM, bool LISTS = false, bool RANGE = false>
__global__ void __launch_bounds__(knn_cfg::NUM_THREADS, 1)
knn_topk_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                const KnnParams p) {
  using namespace knn_cfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  unsigned long long* s_list = reinterpret_cast<unsigned long long*>(smem + STAGES * STAGE_BYTES);  // [64][k]
  unsigned long long* s_queue = s_list + BLOCK_M * MAX_K;                                           // [64][QCAP]
  unsigned long long* s_th = s_queue + BLOCK_M * QCAP;                                              // [64]
  int* s_cnt = reinterpret_cast<int*>(s_th + BLOCK_M);                                              // [64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_cnt + BLOCK_M);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int k = p.k;
  const int64_t row0 = STREAM ? p.row0 : RANGE ? p.row0 : 0;
  IvfItem item = {0, 0, 0, 0, 0};
  if (LISTS) item = p.items[blockIdx.x];
  const int qb = blockIdx.x % p.query_blocks, stripe = LISTS ? item.stripe : blockIdx.x / p.query_blocks;
  const int q0 = LISTS ? item.g0 : qb * BLOCK_M;
  const int q_end = LISTS ? item.g1 : p.Q;
  const int64_t c0 = LISTS ? item.r0 : 0;       // the column of tile 0
  const int64_t c_end = LISTS ? item.r1 : p.N;  // columns >= c_end are no candidates
  const int tiles = LISTS ? (item.r1 - item.r0 + BLOCK_N - 1) / BLOCK_N : (int)((p.N + BLOCK_N - 1) / BLOCK_N);
  const int t_begin = LISTS ? 0 : stripe * p.tiles_per_stripe;
  const int t_end = LISTS ? tiles : min(tiles, t_begin + p.tiles_per_stripe);
  const int num_kb = p.D / BLOCK_K;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_x);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 1);
    }
    fence_barrier_init();
  }
  if constexpr (RANGE) {
    for (int i = threadIdx.x; i < BLOCK_M; i += NUM_THREADS) {  // tau is never NaN: ord(tau) > 0, th does not wrap
      s_th[i] = q0 + i < p.Q ? knn_key(__ldg(p.tau + q0 + i) + 0.0f, 0xFFFFFFFFll) - 1ull : 0ull;
      s_cnt[i] = 0;
    }
  } else {
    for (int i = threadIdx.x; i < BLOCK_M * MAX_K; i += NUM_THREADS) s_list[i] = 0ull;
    for (int i = threadIdx.x; i < BLOCK_M; i += NUM_THREADS) {
      s_th[i] = (STREAM && p.seed != nullptr && q0 + i < p.Q) ? p.seed[(size_t)(q0 + i) * k + k - 1] : 0ull;
      s_cnt[i] = 0;
    }
  }
  __syncthreads();

  const uint32_t wg = __shfl_sync(0xffffffffu, threadIdx.x / 128, 0);
  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (int t = t_begin; t < t_end; ++t) {
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const uint32_t s = it % STAGES;
          while (!mbar_try_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1)) __nanosleep(64);
          mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
          tma_load_2d(smem_a + s * A_STAGE_BYTES, &tmap_q, &full_bar[s], kb * BLOCK_K, q0);
          tma_load_2d(smem_b + s * B_STAGE_BYTES, &tmap_x, &full_bar[s], kb * BLOCK_K, (int)c0 + t * BLOCK_N);
        }
      }
    }
    return;
  }

  // ===================== MMA + top-k warpgroup =====================
  const uint32_t warp = (threadIdx.x / 32) % 4;  // rows [16 warp, +16) of the block
  const uint32_t lane = threadIdx.x % 32;
  const uint32_t g = lane / 4, c = lane % 4;
  const bool signal = (threadIdx.x % 128) == 0;
  const uint32_t a_base = smem_u32(smem_a);
  const uint32_t b_base = smem_u32(smem_b);
  uint32_t it = 0;
  float acc[128];

  int rl[2];           // the thread's rows of the block
  bool rvalid[2];
  int64_t excl[2];     // the excluded column of each row, chunk-local (negative: none); LISTS: the excluded id
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    rl[hr] = (int)(warp * 16 + g + 8 * hr);
    const int q = q0 + rl[hr];
    rvalid[hr] = q < q_end;
    if (LISTS)
      excl[hr] = (p.gself != nullptr && rvalid[hr]) ? p.gself[q] : -1;
    else
      excl[hr] = p.self_offset >= 0 ? (int64_t)q + p.self_offset - row0 : -1;
  }

  // every row's queue into its list: warp w takes rows 16 w .. 16 w + 15
  auto merge_all = [&]() {
    for (int r = (int)warp * 16; r < (int)warp * 16 + 16; ++r)
      if (s_cnt[r] > 0) knn_merge_row<STREAM>(s_list + r * MAX_K, s_queue + r * QCAP, s_cnt + r, s_th + r, k, lane);
  };
  // RANGE: every row's queue appended to the global hit buffer, with one atomicAdd per row for its space
  auto flush_all = [&]() {
    for (int r = (int)warp * 16; r < (int)warp * 16 + 16; ++r) {
      const int n = s_cnt[r];  // warp-uniform, at most QCAP
      if (n == 0) continue;
      unsigned long long at = 0;
      if (lane == 0) {
        at = atomicAdd(p.hit_total, (unsigned long long)n);
        atomicAdd(p.hit_counts + q0 + r, (unsigned long long)n);
      }
      at = __shfl_sync(0xffffffffu, at, 0);
      for (int i = (int)lane; i < n; i += 32)
        if (at + i < (unsigned long long)p.hit_cap) {  // past the capacity the hits are counted, not written
          p.hit_keys[at + i] = s_queue[r * QCAP + i];
          p.hit_rows[at + i] = q0 + r;
        }
      __syncwarp();
      if (lane == 0) s_cnt[r] = 0;
      __syncwarp();
    }
  };

  for (int t = t_begin; t < t_end; ++t) {
    const int64_t n0 = c0 + (int64_t)t * BLOCK_N;
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const uint32_t s = it % STAGES;
      // plain try_wait loop: any call in a wgmma kernel makes ptxas serialise every wgmma (C7510)
      while (!mbar_try_wait(&full_bar[s], (it / STAGES) & 1)) {
      }
      wgmma_fence();
      const uint64_t da = wgmma_desc_sw128(a_base + s * A_STAGE_BYTES);
      const uint64_t db = wgmma_desc_sw128(b_base + s * B_STAGE_BYTES);
#pragma unroll
      for (int kk = 0; kk < BLOCK_K / 16; ++kk) wgmma_m64n256k16(acc, da + 2 * kk, db + 2 * kk, (kb | kk) != 0);
      wgmma_commit();
      wgmma_wait<1>();
      if (kb > 0 && signal) mbar_arrive(&empty_bar[(it + STAGES - 1) % STAGES]);
    }
    wgmma_wait<0>();
    reg_fence_f(acc);
    if (signal) mbar_arrive(&empty_bar[(it + STAGES - 1) % STAGES]);

    // ---- epilogue: acc[4 i + 2 hr + e] is row rl[hr], column n0 + 8 i + 2 c + e.  Thresholds change only in merges,
    // which are bracketed by warpgroup barriers, so each pass reads them fresh.
    // s + 0: a score of -0 becomes +0, so equal scores have equal keys
    bool any = false;
    {
      const unsigned long long th0 = s_th[rl[0]], th1 = s_th[rl[1]];
#pragma unroll
      for (int i = 0; i < 32; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int64_t j = n0 + 8 * i + 2 * (int)c + e;
          if (LISTS) {  // index 0 gives a score's largest key: a superset of the survivors, without reading ids
            const float b = (p.beta != nullptr && j < c_end) ? __ldg(p.beta + j) : 0.f;
            const bool in = j < c_end;
            any |= in && rvalid[0] && knn_key(fmaf(p.alpha, acc[4 * i + e], b) + 0.0f, 0) > th0;
            any |= in && rvalid[1] && knn_key(fmaf(p.alpha, acc[4 * i + 2 + e], b) + 0.0f, 0) > th1;
            continue;
          }
          const float b = (p.beta != nullptr && j < p.N) ? __ldg(p.beta + j) : 0.f;
          const bool in = j < p.N;
          any |= in && rvalid[0] && j != excl[0] && knn_key(fmaf(p.alpha, acc[4 * i + e], b) + 0.0f, j + row0) > th0;
          any |= in && rvalid[1] && j != excl[1] &&
                 knn_key(fmaf(p.alpha, acc[4 * i + 2 + e], b) + 0.0f, j + row0) > th1;
        }
      }
    }
    if (!knn_bar_or(1, any)) continue;
#pragma unroll
    for (int ch = 0; ch < BLOCK_N / CHUNK; ++ch) {
      const unsigned long long th0 = s_th[rl[0]], th1 = s_th[rl[1]];
      bool full = false;
#pragma unroll
      for (int ii = 0; ii < CHUNK / 8; ++ii) {
        const int i = ch * (CHUNK / 8) + ii;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int64_t j = n0 + 8 * i + 2 * (int)c + e;
          if (LISTS) {  // ids[j] is read only for a score that can pass the threshold
            const float b = (p.beta != nullptr && j < c_end) ? __ldg(p.beta + j) : 0.f;
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const float sc = fmaf(p.alpha, acc[4 * i + 2 * hr + e], b) + 0.0f;
              const unsigned long long th = hr ? th1 : th0;
              if (j < c_end && rvalid[hr] && knn_key(sc, 0) > th) {
                const int64_t id = __ldg(reinterpret_cast<const long long*>(p.ids) + j);
                const unsigned long long key = knn_key(sc, id);
                if (id != excl[hr] && key > th) {
                  const int pos = atomicAdd(s_cnt + rl[hr], 1);
                  s_queue[rl[hr] * QCAP + pos] = key;
                  full |= pos >= QCAP - CHUNK;
                }
              }
            }
            continue;
          }
          const float b = (p.beta != nullptr && j < p.N) ? __ldg(p.beta + j) : 0.f;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const unsigned long long key = knn_key(fmaf(p.alpha, acc[4 * i + 2 * hr + e], b) + 0.0f, j + row0);
            if (j < p.N && rvalid[hr] && j != excl[hr] && key > (hr ? th1 : th0)) {
              const int pos = atomicAdd(s_cnt + rl[hr], 1);  // < QCAP: at most QCAP - CHUNK queued before a chunk
              s_queue[rl[hr] * QCAP + pos] = key;
              full |= pos >= QCAP - CHUNK;
            }
          }
        }
      }
      if (knn_bar_or(1, full)) {
        if constexpr (RANGE) flush_all(); else merge_all();
        named_bar_sync(1, 128);
      }
    }
  }
  named_bar_sync(1, 128);
  if constexpr (RANGE) {
    flush_all();
    return;
  }
  merge_all();
  __syncwarp();
  // ---- the stripe's lists: warp w writes rows 16 w ..
  for (int r = (int)warp * 16; r < (int)warp * 16 + 16; ++r) {
    const int q = q0 + r;
    if (q >= q_end) break;
    if (LISTS && p.pbase[q] < 0) continue;
    unsigned long long* dst = LISTS ? p.keys + ((size_t)p.pbase[q] + stripe) * k : p.keys + ((size_t)stripe * p.Q + q) * k;
    for (int i = (int)lane; i < k; i += 32) dst[i] = s_list[r * MAX_K + i];
  }
}

// One block per query: k rounds, each taking the largest head of the lists (keys are distinct, so the winner is unique
// unless it is an empty slot) and advancing that list.  The lists are the S stripe lists and, with ACC, the running
// list run[q] as list S; thread t owns lists t, t + blockDim, ... (at most M).  Without ACC the winners are decoded to
// out_scores / out_idx; with ACC they are written back to run[q] as keys.  RAGGED (esmb200_ivf_search): query q has
// counts[q] lists, at keys[q * S + s] (S the per-query stride), and an empty slot decodes to NaN and index -1.
template <int M, bool ACC, bool RAGGED = false>
__global__ void __launch_bounds__(256)
knn_merge_kernel(const unsigned long long* __restrict__ keys, int Q, int k, int S, unsigned long long* run,
                 float* __restrict__ out_scores, int64_t* __restrict__ out_idx, const int* counts = nullptr) {
  __shared__ unsigned long long red_key[2][8];
  __shared__ int red_s[2][8];
  __shared__ unsigned long long s_run[ACC ? knn_cfg::MAX_K : 1];
  const int q = blockIdx.x;
  const int nt = blockDim.x, warp = threadIdx.x / 32, nw = nt / 32;
  const int L = RAGGED ? counts[q] : ACC ? S + 1 : S;
  if (ACC) {
    for (int i = threadIdx.x; i < k; i += nt) s_run[i] = run[(size_t)q * k + i];
    __syncthreads();
  }
  auto fetch = [&](int s, int pos) -> unsigned long long {
    if (ACC && s == S) return s_run[pos];
    if (RAGGED) return keys[((size_t)q * S + s) * k + pos];
    return keys[((size_t)s * Q + q) * k + pos];
  };
  unsigned long long head[M];
  int pos[M];
#pragma unroll
  for (int m = 0; m < M; ++m) {
    const int s = threadIdx.x + m * nt;
    pos[m] = 0;
    head[m] = s < L ? fetch(s, 0) : 0ull;
  }
  for (int r = 0; r < k; ++r) {
    unsigned long long best = 0ull;
    int bs = -1;
#pragma unroll
    for (int m = 0; m < M; ++m)
      if (head[m] > best || bs < 0) {
        best = head[m];
        bs = threadIdx.x + m * nt;
      }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long b2 = __shfl_xor_sync(0xffffffffu, best, o);
      const int s2 = __shfl_xor_sync(0xffffffffu, bs, o);
      if (b2 > best || (b2 == best && s2 < bs)) {
        best = b2;
        bs = s2;
      }
    }
    if (threadIdx.x % 32 == 0) {
      red_key[r & 1][warp] = best;
      red_s[r & 1][warp] = bs;
    }
    __syncthreads();
    best = red_key[r & 1][0];
    bs = red_s[r & 1][0];
    for (int w = 1; w < nw; ++w) {
      const unsigned long long b2 = red_key[r & 1][w];
      const int s2 = red_s[r & 1][w];
      if (b2 > best || (b2 == best && s2 < bs)) {
        best = b2;
        bs = s2;
      }
    }
#pragma unroll
    for (int m = 0; m < M; ++m)
      if (bs == (int)threadIdx.x + m * nt && bs < L) {
        ++pos[m];
        head[m] = pos[m] < k ? fetch(bs, pos[m]) : 0ull;
      }
    if (threadIdx.x == 0) {
      if (ACC)
        run[(size_t)q * k + r] = best;
      else
        knn_decode_key(best, out_scores + (size_t)q * k + r, out_idx + (size_t)q * k + r);
      if (RAGGED && best == 0ull) out_idx[(size_t)q * k + r] = -1;
    }
  }
}

// keys [n] to fp32 scores and int64 indices, as knn_merge_kernel<M, false> writes them
__global__ void __launch_bounds__(256)
knn_decode_kernel(const unsigned long long* __restrict__ keys, int64_t n, float* __restrict__ out_scores,
                  int64_t* __restrict__ out_idx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    knn_decode_key(keys[i], out_scores + i, out_idx + i);
}

// ---- range search (esmb200_knn_range_finish): the appended hits, sorted by (query row, key descending), to CSR -------
// One block of 1024 threads: off = exclusive scan of counts (where each query's hits start), lims = exclusive scan of
// min(counts, max_hits) (max_hits < 0: no cap); both [Q + 1].
__global__ void __launch_bounds__(1024)
knn_range_scan_kernel(const long long* __restrict__ counts, int Q, long long max_hits, long long* __restrict__ off,
                      long long* __restrict__ lims) {
  __shared__ long long s_o[1024], s_l[1024];
  const int per = (Q + 1023) / 1024, l0 = min(Q, (int)threadIdx.x * per), l1 = min(Q, l0 + per);
  auto kept = [&](long long c) { return max_hits >= 0 && c > max_hits ? max_hits : c; };
  long long so = 0, sl = 0;
  for (int q = l0; q < l1; ++q) {
    so += counts[q];
    sl += kept(counts[q]);
  }
  s_o[threadIdx.x] = so;
  s_l[threadIdx.x] = sl;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long ao = 0, al = 0;
    for (int t = 0; t < 1024; ++t) {
      const long long o = s_o[t], l = s_l[t];
      s_o[t] = ao;
      s_l[t] = al;
      ao += o;
      al += l;
    }
    off[Q] = ao;
    lims[Q] = al;
  }
  __syncthreads();
  so = s_o[threadIdx.x];
  sl = s_l[threadIdx.x];
  for (int q = l0; q < l1; ++q) {
    off[q] = so;
    lims[q] = sl;
    so += counts[q];
    sl += kept(counts[q]);
  }
}

// hit p (query rows[p], rank p - off[q] within its query) goes to lims[q] + rank when the rank is below the query's
// kept count, decoded to a score and an index
__global__ void __launch_bounds__(256)
knn_range_decode_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ rows, int64_t nnz, int Q,
                        const long long* __restrict__ off, const long long* __restrict__ lims,
                        float* __restrict__ out_scores, int64_t* __restrict__ out_idx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
    const int q = rows[i];
    if (q < 0 || q >= Q) continue;
    const long long r = i - off[q];
    if (r < 0 || r >= lims[q + 1] - lims[q]) continue;
    knn_decode_key(keys[i], out_scores + lims[q] + r, out_idx + lims[q] + r);
  }
}

// ---- inverted-file search (esmb200_ivf_search): the grouping of (query, probe) pairs into list-scan work items --------
// A list's stripes: T 256-row tiles each, so S_l = ceil(ceil(len_l / 256) / T).
__device__ __forceinline__ int ivf_stripes(const int64_t* offsets, int l, int64_t N, int T) {
  const int64_t a = min(max(offsets[l], (int64_t)0), N), b = min(max(offsets[l + 1], a), N);
  const int64_t tiles = (b - a + knn_cfg::BLOCK_N - 1) / knn_cfg::BLOCK_N;
  return (int)((tiles + T - 1) / T);
}

// each pair (query, probe) takes the next position in its list's group; an entry outside [0, nlist), or one that
// repeats an earlier entry of its row, probes nothing (slot -1), so a list is scanned at most once per query.  The
// positions depend on the order the atomics land in, which changes no result: the top k under the key order does not
// depend on the order candidates are seen in.
__global__ void __launch_bounds__(256)
ivf_count_kernel(const int32_t* __restrict__ probes, int64_t P, int nprobe, int nlist, int* __restrict__ cnt,
                 int* __restrict__ slot) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = probes[i];
    bool ok = l >= 0 && l < nlist;
    for (int64_t j = i - i % nprobe; ok && j < i; ++j) ok = probes[j] != l;
    slot[i] = ok ? atomicAdd(cnt + l, 1) : -1;
  }
}

// one block of 512 threads: gstart = exclusive scan of the group sizes, istart = exclusive scan of the work items per list
// (ceil(cnt / 64) query blocks times the list's stripes); both [nlist + 1]
__global__ void __launch_bounds__(512)
ivf_scan_kernel(const int* __restrict__ cnt, const int64_t* __restrict__ offsets, int nlist, int64_t N, int T,
                int* __restrict__ gstart, int* __restrict__ istart) {
  __shared__ int s_g[512], s_i[512];
  const int per = (nlist + 511) / 512, l0 = threadIdx.x * per, l1 = min(nlist, l0 + per);
  int sg = 0, si = 0;
  for (int l = l0; l < l1; ++l) {
    sg += cnt[l];
    si += (cnt[l] + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M * ivf_stripes(offsets, l, N, T);
  }
  s_g[threadIdx.x] = sg;
  s_i[threadIdx.x] = si;
  __syncthreads();
  if (threadIdx.x == 0) {
    int ag = 0, ai = 0;
    for (int t = 0; t < 512; ++t) {
      const int g = s_g[t], i = s_i[t];
      s_g[t] = ag;
      s_i[t] = ai;
      ag += g;
      ai += i;
    }
    gstart[nlist] = ag;
    istart[nlist] = ai;
  }
  __syncthreads();
  sg = s_g[threadIdx.x];
  si = s_i[threadIdx.x];
  for (int l = l0; l < l1; ++l) {
    gstart[l] = sg;
    istart[l] = si;
    sg += cnt[l];
    si += (cnt[l] + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M * ivf_stripes(offsets, l, N, T);
  }
}

// one thread per query: its gathered rows (query index, excluded id) and their partial lists, R per query, in probe
// order; counts[q] = the query's partial lists.  A pair whose stripes would pass R (only with offsets that do not
// partition [0, N)) writes nothing.
__global__ void __launch_bounds__(256)
ivf_place_kernel(const int32_t* __restrict__ probes, const int* __restrict__ slot, const int* __restrict__ gstart,
                 const int64_t* __restrict__ offsets, int Q, int nprobe, int nlist, int64_t N, int T, int R,
                 const int64_t* __restrict__ self_ids, int* __restrict__ gq, int64_t* __restrict__ gself,
                 int* __restrict__ pbase, int* __restrict__ counts) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  int run = 0;
  for (int i = 0; i < nprobe; ++i) {
    const int64_t pr = (int64_t)q * nprobe + i;
    const int l = probes[pr];
    if (slot[pr] < 0) continue;
    const int g = gstart[l] + slot[pr], S = ivf_stripes(offsets, l, N, T);
    gq[g] = q;
    gself[g] = self_ids != nullptr ? self_ids[q] : -1;
    pbase[g] = run + S <= R ? q * R + run : -1;
    run += run + S <= R ? S : 0;
  }
  counts[q] = run;
}

// one thread per list: its work items, query block major, at istart[l]
__global__ void __launch_bounds__(256)
ivf_items_kernel(const int* __restrict__ cnt, const int* __restrict__ gstart, const int* __restrict__ istart,
                 const int64_t* __restrict__ offsets, int nlist, int64_t N, int T, IvfItem* __restrict__ items) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= nlist) return;
  const int S = ivf_stripes(offsets, l, N, T), nb = (cnt[l] + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M;
  const int64_t a = min(max(offsets[l], (int64_t)0), N), b = min(max(offsets[l + 1], a), N);
  const int64_t span = (int64_t)T * knn_cfg::BLOCK_N;
  for (int qb = 0; qb < nb; ++qb)
    for (int s = 0; s < S; ++s) {
      IvfItem it;
      it.g0 = gstart[l] + qb * knn_cfg::BLOCK_M;
      it.g1 = min(gstart[l] + cnt[l], it.g0 + knn_cfg::BLOCK_M);
      it.r0 = (int)(a + s * span);
      it.r1 = (int)min(b, a + (s + 1) * span);
      it.stripe = s;
      items[istart[l] + qb * S + s] = it;
    }
}

// every list at once (nprobe == nlist): the stored rows in S stripes of T tiles, stripe major as knn_topk_kernel's
// grid, and each query's S partial lists at q * S
__global__ void __launch_bounds__(256)
ivf_all_items_kernel(int Q, int64_t N, int S, int T, IvfItem* __restrict__ items, int* __restrict__ pbase,
                     int* __restrict__ counts) {
  const int blocks = (Q + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M;
  const int64_t span = (int64_t)T * knn_cfg::BLOCK_N;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < blocks * S; i += gridDim.x * blockDim.x) {
    const int qb = i % blocks, s = i / blocks;
    IvfItem it;
    it.g0 = qb * knn_cfg::BLOCK_M;
    it.g1 = min(Q, it.g0 + knn_cfg::BLOCK_M);
    it.r0 = (int)min(N, s * span);
    it.r1 = (int)min(N, (s + 1) * span);
    it.stripe = s;
    items[i] = it;
  }
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < Q; q += gridDim.x * blockDim.x) {
    pbase[q] = q * S;
    counts[q] = S;
  }
}

// gathered query rows: dst [P, D] (dense) row g = src row gq[g] for the *placed rows (pairs with a list); 16-byte copies
__global__ void __launch_bounds__(256)
ivf_gather_kernel(const __half* __restrict__ src, int64_t ld, const int* __restrict__ gq, const int* __restrict__ placed,
                  int D, __half* __restrict__ dst) {
  const int per = D / 8;
  const int64_t P = *placed;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < P * per; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = i / per;
    const int c = (int)(i % per);
    reinterpret_cast<uint4*>(dst + g * D)[c] = reinterpret_cast<const uint4*>(src + (int64_t)gq[g] * ld)[c];
  }
}

// ---- k-means means (esmb200_kmeans_means) ---------------------------------------------------------------------------
// Every fp16 value is an integer multiple of 2^-24, so x * 2^24 is an exact integer and the member sum per column is
// an exact int64 whatever order the atomics land in.  One warp per row.
__global__ void __launch_bounds__(256)
kmeans_sum_kernel(const __half* __restrict__ rows, int64_t ld, int64_t n, int D, const int64_t* __restrict__ assign,
                  int nlist, unsigned long long* __restrict__ sums, unsigned long long* __restrict__ counts) {
  const int lane = threadIdx.x % 32;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x / 32);
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; r < n; r += warps) {
    const int64_t c = assign[r];
    if (c < 0 || c >= nlist) continue;
    if (lane == 0) atomicAdd(counts + c, 1ull);
    for (int v = lane; v < D / 8; v += 32) {
      const uint4 u = reinterpret_cast<const uint4*>(rows + r * ld)[v];
      const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const long long x = __float2ll_rn(__half2float(h[e]) * 16777216.0f);
        if (x != 0) atomicAdd(sums + c * D + 8 * v + e, (unsigned long long)x);
      }
    }
  }
}

// means[c, j] = fp32(((double)S / count) * 2^-24), 0 for an empty cluster
__global__ void __launch_bounds__(256)
kmeans_mean_kernel(const long long* __restrict__ sums, const long long* __restrict__ counts, int nlist, int D,
                   float* __restrict__ means) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)nlist * D;
       i += (int64_t)gridDim.x * blockDim.x) {
    const long long cnt = counts[i / D];
    means[i] = cnt > 0 ? __double2float_rn(__ddiv_rn((double)sums[i], (double)cnt) * 0x1p-24) : 0.f;
  }
}

}  // namespace esmb200
