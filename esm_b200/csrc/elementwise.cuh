// esm_b200 — HBM-bound row kernels around the tensor-core GEMMs (sm_90a).
//
//   layernorm_rows    esm/modules.py:68-81,124,137 and esm/model/esm2.py:123 (torch.nn.LayerNorm, eps 1e-5, affine),
//                     one warp per row, the row held in registers (single HBM read), fp16 or fp32 output
//   embed_tokens      esm/model/esm2.py:84-95 (embedding gather, <mask> zeroing, token-dropout rescale
//                     0.88/(1-mask_ratio), pad zeroing)
//   esm1b_embed       esm/model/esm1.py:121-139 (the same, plus learned positions and emb_layer_norm_before)
//   key_bits          esm/model/esm2.py:82 + multihead_attention.py:368-374 (key padding mask) packed to 1 bit/key
//   mean_pool         scripts/extract.py:116-119 per-sequence mean representation
//   log_softmax_rows  examples/variant-prediction/predict.py:142,175,194,211 (torch.log_softmax over the vocabulary)
//                     and the target gather of :114,143
//   window_merge      weighted row sums that stitch overlapping windows of a long protein (esm_b200/windows.py)
//   convert_f32_f16   weight packing (fp32 nn.Linear weights -> fp16 MMA operands)
#pragma once

#include "common.cuh"

namespace esmb200 {

// Each lane owns float4 chunks lane, lane+32, ... of the row. MAXV bounds E <= MAXV*128.
// OUT: 0 = fp32 [M,E]; 1 = fp16 [M,E] (GEMM A operand); 2 = fp16 hi | lo [M,2E] (A operand of the fp32x3 GEMMs:
// hi = rn(y) in columns [0,E), lo = rn(y - hi) in columns [E,2E)); 3 = e4m3 [M,E] and one power-of-two scale per row
// and 128 columns, scales[kb * M + row] (A operand of the fp8 GEMMs: a lane's float4 chunk i lies in 128-column block i,
// so a block's amax is one warp reduction).
template <int MAXV, int OUT>
__global__ void __launch_bounds__(256)
layernorm_rows_kernel(const float* x, const float* __restrict__ gamma, const float* __restrict__ beta, void* out, int M,
                      int E, float eps, float* scales) {  // x and out may alias (in-place final LayerNorm): a warp reads its whole row first
  const int warps_per_block = blockDim.x / 32;
  const int row = blockIdx.x * warps_per_block + threadIdx.x / 32;
  if (row >= M) return;
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x % 32;
  const int nvec = E / 4;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * E);
  float4 v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      v[i] = xr[idx];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mean = warp_sum(s) / (float)E;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)E + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  if constexpr (OUT == 3) {
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      if (i * 128 >= E) break;  // warp-uniform: every lane takes part in the block's reduction
      const int idx = lane + i * 32;
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < nvec) {
        const float4 g = __ldg(g4 + idx), b = __ldg(b4 + idx);
        o.x = (v[i].x - mean) * rstd * g.x + b.x;
        o.y = (v[i].y - mean) * rstd * g.y + b.y;
        o.z = (v[i].z - mean) * rstd * g.z + b.z;
        o.w = (v[i].w - mean) * rstd * g.w + b.w;
      }
      const float sc = fp8_block_scale(warp_max(fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w)))));
      const float inv = __frcp_rn(sc);  // o * inv == o / sc exactly
      if (idx < nvec)
        reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(out) + (size_t)row * E)[idx] =
            (uint32_t)cvt_e4m3x2(o.x * inv, o.y * inv) | ((uint32_t)cvt_e4m3x2(o.z * inv, o.w * inv) << 16);
      if (lane == 0) scales[(size_t)i * M + row] = sc;
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      const float4 g = __ldg(g4 + idx), b = __ldg(b4 + idx);
      float4 o;
      o.x = (v[i].x - mean) * rstd * g.x + b.x;
      o.y = (v[i].y - mean) * rstd * g.y + b.y;
      o.z = (v[i].z - mean) * rstd * g.z + b.z;
      o.w = (v[i].w - mean) * rstd * g.w + b.w;
      if constexpr (OUT == 1) {
        uint2 h;
        h.x = pack_half2(o.x, o.y);
        h.y = pack_half2(o.z, o.w);
        reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out) + (size_t)row * E)[idx] = h;
      } else if constexpr (OUT == 2) {
        const __half2 h01 = __floats2half2_rn(o.x, o.y), h23 = __floats2half2_rn(o.z, o.w);
        const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
        uint2 h, l;
        h.x = *reinterpret_cast<const uint32_t*>(&h01);
        h.y = *reinterpret_cast<const uint32_t*>(&h23);
        l.x = pack_half2(o.x - f01.x, o.y - f01.y);
        l.y = pack_half2(o.z - f23.x, o.w - f23.y);
        __half* orow = reinterpret_cast<__half*>(out) + (size_t)row * 2 * E;
        reinterpret_cast<uint2*>(orow)[idx] = h;
        reinterpret_cast<uint2*>(orow + E)[idx] = l;
      } else {
        reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + (size_t)row * E)[idx] = o;
      }
    }
  }
}

template <int OUT>
inline cudaError_t launch_layernorm(const float* x, const float* gamma, const float* beta, void* out, int M, int E,
                                    float eps, cudaStream_t stream, float* scales = nullptr) {
  if (E % 4 != 0 || E > 40 * 128) return cudaErrorInvalidValue;
  const int wpb = 8;
  const int grid = (M + wpb - 1) / wpb;
  if (grid == 0) return cudaSuccess;
  const dim3 g(grid), b(wpb * 32);
  if (E <= 4 * 128) return launch_pdl(layernorm_rows_kernel<4, OUT>, g, b, 0, stream, x, gamma, beta, out, M, E, eps,
                                         scales);
  if (E <= 10 * 128) return launch_pdl(layernorm_rows_kernel<10, OUT>, g, b, 0, stream, x, gamma, beta, out, M, E, eps,
                                         scales);
  if (E <= 20 * 128) return launch_pdl(layernorm_rows_kernel<20, OUT>, g, b, 0, stream, x, gamma, beta, out, M, E, eps,
                                         scales);
  return launch_pdl(layernorm_rows_kernel<40, OUT>, g, b, 0, stream, x, gamma, beta, out, M, E, eps, scales);
}

// grid (row chunks, B): every block counts the <mask>/<pad> tokens of its sequence (T 8-byte reads, cheaper than a
// separate pass) and writes the scaled embedding rows of its chunk.  (One block per sequence left a 32-sequence batch —
// the per-GPU share at 8 GPUs — on 32 SMs: 0.6 ms, 1 % of that step.)
__global__ void __launch_bounds__(256)
embed_tokens_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ table, float* __restrict__ x, int T,
                    int E, int padding_idx, int mask_idx, int token_dropout) {
  const int b = blockIdx.y;
  const int64_t* tok = tokens + (size_t)b * T;
  __shared__ int s_cnt[2];
  if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  if (token_dropout) {
    int n_mask = 0, n_pad = 0;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
      const int64_t v = tok[t];
      n_mask += (v == mask_idx);
      n_pad += (v == padding_idx);
    }
    n_mask = (int)warp_sum((float)n_mask);
    n_pad = (int)warp_sum((float)n_pad);
    if (threadIdx.x % 32 == 0) {
      atomicAdd(&s_cnt[0], n_mask);
      atomicAdd(&s_cnt[1], n_pad);
    }
    __syncthreads();
  }
  // esm2.py:86-92: x.masked_fill_(mask, 0); x = x * (1 - 0.15*0.8) / (1 - n_mask / src_length)
  // (python evaluates 1 - 0.15*0.8 in double, the tensor ops run in fp32: multiply first, then divide)
  const float keep = (float)(1.0 - 0.15 * 0.8);
  const float denom = 1.0f - (float)s_cnt[0] / (float)(T - s_cnt[1]);
  const int nvec = E / 4;
  const int rows = (T + gridDim.x - 1) / gridDim.x;
  const int t0 = blockIdx.x * rows, t1 = min(T, t0 + rows);
  for (int i = t0 * nvec + threadIdx.x; i < t1 * nvec; i += blockDim.x) {
    const int t = i / nvec, c = i % nvec;
    const int64_t v = tok[t];
    float4 e = __ldg(reinterpret_cast<const float4*>(table + (size_t)v * E) + c);
    if (token_dropout) {
      if (v == mask_idx) e = make_float4(0.f, 0.f, 0.f, 0.f);
      e.x = (e.x * keep) / denom;
      e.y = (e.y * keep) / denom;
      e.z = (e.z * keep) / denom;
      e.w = (e.w * keep) / denom;
    }
    if (v == padding_idx) e = make_float4(0.f, 0.f, 0.f, 0.f);
    reinterpret_cast<float4*>(x + ((size_t)b * T + t) * E)[c] = e;
  }
}

// keybits[b, w] bit i = key 32w+i attendable; kvlen[b] = 1 + last attendable key. One warp per sequence.
__global__ void key_bits_kernel(const uint8_t* __restrict__ pad_mask, uint32_t* __restrict__ keybits,
                                int* __restrict__ kvlen, int B, int T, int words) {
  const int b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (b >= B) return;
  const int lane = threadIdx.x % 32;
  int last = 0;
  for (int w = 0; w < words; ++w) {
    const int key = w * 32 + lane;
    bool ok = key < T;
    if (ok && pad_mask) ok = pad_mask[(size_t)b * T + key] == 0;
    const uint32_t bits = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) keybits[(size_t)b * words + w] = bits;
    if (bits) last = w * 32 + (32 - __clz(bits));
  }
  if (lane == 0) kvlen[b] = last;
}

// Per-sequence mean over residues (scripts/extract.py:116-119: representations[i, 1 : len+1].mean(0)).
// grid (ceil(E/128), B), block 256 = 8 row lanes x 32 float4 columns: row lane r sums the residues t = r (mod 8) of its
// 128 columns (512-byte coalesced warp rows, 4 independent accumulators), the 8 partial sums are combined through shared
// memory in a fixed order (deterministic).  E % 4 == 0.
__global__ void __launch_bounds__(256)
mean_pool_kernel(const float* __restrict__ x, const int* __restrict__ lengths, float* __restrict__ out, int T, int E) {
  const int b = blockIdx.y;
  const int lane = threadIdx.x % 32, rl = threadIdx.x / 32;
  const int col = blockIdx.x * 128 + lane * 4;
  __shared__ float4 part[8][32];
  int n = lengths[b];
  n = n < 0 ? 0 : (n > T - 1 ? T - 1 : n);
  float4 a[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) a[u] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (col < E) {
    const float* xp = x + ((size_t)b * T + 1) * E + col;
    int t = rl;
    for (; t + 24 < n; t += 32) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float4 v = *reinterpret_cast<const float4*>(xp + (size_t)(t + 8 * u) * E);
        a[u].x += v.x; a[u].y += v.y; a[u].z += v.z; a[u].w += v.w;
      }
    }
    for (; t < n; t += 8) {
      const float4 v = *reinterpret_cast<const float4*>(xp + (size_t)t * E);
      a[0].x += v.x; a[0].y += v.y; a[0].z += v.z; a[0].w += v.w;
    }
  }
  part[rl][lane] = make_float4((a[0].x + a[1].x) + (a[2].x + a[3].x), (a[0].y + a[1].y) + (a[2].y + a[3].y),
                               (a[0].z + a[1].z) + (a[2].z + a[3].z), (a[0].w + a[1].w) + (a[2].w + a[3].w));
  __syncthreads();
  if (rl == 0 && col < E) {
    float4 s = part[0][lane];
#pragma unroll
    for (int r = 1; r < 8; ++r) {
      const float4 v = part[r][lane];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    const float inv = 1.0f / (float)n;  // n == 0: inf * 0 = NaN like the reference's mean over an empty slice
    *reinterpret_cast<float4*>(out + (size_t)b * E + col) = make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv);
  }
}

// Row max m and lse = logf(sum of expf(x - m)) of a row of at most 64 columns held by one warp, lane l holding
// columns l (v0) and l + 32 (v1), -INFINITY past the row's end. The arithmetic follows PyTorch's warp-per-row softmax:
// row max, per-lane sum in column order, xor-butterfly sums. expf / logf are the accurate library functions, not
// ex2.approx. Every lane gets m and lse.
__device__ __forceinline__ void warp_row_lse(float v0, float v1, float& m, float& lse) {
  m = fmaxf(v0, v1);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = expf(v0 - m);
  s += expf(v1 - m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  lse = logf(s);
}

// log_softmax over the first V <= 64 columns of each row: one warp per row (warp_row_lse), then (x - max) - lse.
// target == nullptr: out [n, V]; otherwise out[i] = the value of column target[i] (in [0, V), checked by the caller).
__global__ void __launch_bounds__(256)
log_softmax_rows_kernel(const float* __restrict__ logits, int64_t ld, int n, int V, const int64_t* __restrict__ target,
                        float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= n) return;
  const float* x = logits + (size_t)row * ld;
  const float v0 = lane < V ? x[lane] : -INFINITY;
  const float v1 = lane + 32 < V ? x[lane + 32] : -INFINITY;
  float m, lse;
  warp_row_lse(v0, v1, m, lse);
  if (target) {
    if (lane == 0) out[row] = (x[target[row]] - m) - lse;
  } else {
    float* y = out + (size_t)row * V;
    if (lane < V) y[lane] = (v0 - m) - lse;
    if (lane + 32 < V) y[lane + 32] = (v1 - m) - lse;
  }
}

// Overlapping-window merge (esm_b200/windows.py): out[r, c] = sum over j in [seg[r], seg[r+1]) of w[j] * src[idx[j], c].
// One thread per output element (flat r * C + c, so neighbouring threads read neighbouring columns of a source row for
// any C), grid-stride. The terms are taken in j order as one fp32 fma chain; a one-term segment is a plain copy (every
// bit pattern, -0.0 and NaN included, passes through), an empty one writes +0. No atomics: deterministic.
__global__ void __launch_bounds__(256)
window_merge_kernel(const float* __restrict__ src, int64_t src_ld, const int64_t* __restrict__ idx,
                    const float* __restrict__ w, const int64_t* __restrict__ seg, int64_t rows, int C,
                    float* __restrict__ out, int64_t out_ld) {
  const int64_t total = rows * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C;
    const int c = (int)(i - r * C);
    const int64_t j0 = seg[r], j1 = seg[r + 1];
    float acc = 0.f;
    if (j1 - j0 == 1) {
      acc = src[idx[j0] * src_ld + c];
    } else {
      for (int64_t j = j0; j < j1; ++j) acc = fmaf(w[j], src[idx[j] * src_ld + c], acc);
    }
    out[r * out_ld + c] = acc;
  }
}

__global__ void convert_f32_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) dst[i] = __float2half_rn(src[i]);
}

// fp32x3 operands: src [rows, K] fp32 -> dst [rows, 2K] fp16, hi = rn(x) in columns [0,K), lo = rn(x - hi) in [K,2K)
__global__ void convert_f32_split_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t rows, int K) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n = rows * (size_t)K, stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const size_t r = i / K, k = i % K;
    const float x = src[i];
    const __half h = __float2half_rn(x);
    dst[r * 2 * K + k] = h;
    dst[r * 2 * K + K + k] = __float2half_rn(x - __half2float(h));
  }
}

// head_dim != 64: every head's projection rows go to zero-padded 64-wide *slots* — one per head for d <= 64, two for
// 64 < d <= 128 (ESM-2 15B).  The reference's rotate-half pair p = (j, j + d/2), p < d/2 (rotary_embedding.py:11-20),
// lands in slot p / 32 at positions (p % 32, 32 + p % 32), so the RoPE epilogue's fixed (c, c + 32) pairing inside a
// 64-column group reproduces it with table column p, and q.k / P.v — sums over the head dimension — do not care about the
// order.  dst must be zero-filled by the caller.
__device__ __forceinline__ int head_slot(int n, int d) {  // projection output index n = h*d + j -> attention-side column
  const int h = n / d, j = n % d, half = d / 2;
  const int pr = j < half ? j : j - half;
  const int slots = d > 64 ? 2 : 1;
  return (h * slots + pr / 32) * 64 + (pr % 32) + (j < half ? 0 : 32);
}
// split != 0: fp32x3 operand layout, row pitch 2K with the lo halves K columns to the right
__global__ void pack_head_rows_kernel(const float* __restrict__ w, const float* __restrict__ b, __half* __restrict__ dst,
                                      float* __restrict__ bdst, int E, int d, int split) {  // w [E,E] -> dst [Ea, E]
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)E * E) return;
  const int n = (int)(i / E), k = (int)(i % E);
  const int r = head_slot(n, d);
  const __half h = __float2half_rn(w[i]);
  const size_t pitch = split ? 2 * (size_t)E : (size_t)E;
  dst[(size_t)r * pitch + k] = h;
  if (split) dst[(size_t)r * pitch + E + k] = __float2half_rn(w[i] - __half2float(h));
  if (k == 0) bdst[r] = b[n];
}
__global__ void pack_head_cols_kernel(const float* __restrict__ w, __half* __restrict__ dst, int E, int Ea, int d,
                                      int split) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // w [E,E] (out_proj) -> dst [E, Ea]
  if (i >= (size_t)E * E) return;
  const int n = (int)(i / E), k = (int)(i % E);
  const __half h = __float2half_rn(w[i]);
  const size_t pitch = split ? 2 * (size_t)Ea : (size_t)Ea;
  dst[(size_t)n * pitch + head_slot(k, d)] = h;
  if (split) dst[(size_t)n * pitch + Ea + head_slot(k, d)] = __float2half_rn(w[i] - __half2float(h));
}

// fp8 precision: the QKV weight rows in their head slots as fp32 (w [E,E] -> dst [Ea, E], zero-filled by the caller), so
// that the 128 x 128 block quantisation sees exactly the fp32 weights
__global__ void pack_head_rows_f32_kernel(const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ dst,
                                          float* __restrict__ bdst, int E, int d) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)E * E) return;
  const int n = (int)(i / E), k = (int)(i % E);
  const int r = head_slot(n, d);
  dst[(size_t)r * E + k] = w[i];
  if (k == 0) bdst[r] = b[n];
}

// fp32 [rows, K] -> e4m3 [rows, K], one power-of-two scale (fp8_block_scale) per block of block_rows x 128 columns:
// block_rows 1 (activations; scales [ceil(K/128), rows]) or 128 (weights; scales [ceil(rows/128), ceil(K/128)]).
// A partial block takes its scale over its valid elements.  Grid (ceil(K/128), ceil(rows/block_rows)), 256 threads.
__global__ void __launch_bounds__(256)
quantize_fp8_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst, float* __restrict__ scales, int rows, int K,
                    int block_rows) {
  __shared__ float red[8];
  const int kb = blockIdx.x, r_lo = blockIdx.y * block_rows, k0 = kb * 128;
  const int nr = min(block_rows, rows - r_lo), nk = min(128, K - k0);
  float m = 0.f;
  for (int e = threadIdx.x; e < nr * 128; e += 256)
    if (e % 128 < nk) m = fmaxf(m, fabsf(src[(size_t)(r_lo + e / 128) * K + k0 + e % 128]));
  m = warp_max(m);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = m;
  __syncthreads();
  m = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) m = fmaxf(m, red[w]);
  const float sc = fp8_block_scale(m), inv = __frcp_rn(sc);
  for (int e = threadIdx.x; e < nr * 128; e += 256)
    if (e % 128 < nk) {
      const size_t at = (size_t)(r_lo + e / 128) * K + k0 + e % 128;
      dst[at] = (uint8_t)(cvt_e4m3x2(src[at] * inv, 0.f) & 0xffu);
    }
  if (threadIdx.x == 0) scales[block_rows == 1 ? (size_t)kb * rows + r_lo : (size_t)blockIdx.y * gridDim.x + kb] = sc;
}

// MSA row attention: q is zeroed at padded positions before the logits are summed over the alignment rows
// (/root/reference/esm/axial_attention.py:82-85).  qkv [M, 3E] fp16, pad [M] (1 = padding); one warp per row.
// SPLIT (fp32x3): qkv [M, 6E] = [q k v]_hi | [q k v]_lo, and q_lo (columns [3E, 4E)) is zeroed as well.
template <bool SPLIT>
__global__ void __launch_bounds__(256)
zero_q_at_pads_kernel(__half* __restrict__ qkv, const uint8_t* __restrict__ pad, int M, int E) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * 8 + threadIdx.x / 32;
  if (row >= M || !pad[row]) return;
  uint4* q = reinterpret_cast<uint4*>(qkv + (size_t)row * (SPLIT ? 6 : 3) * E);  // E % 64 == 0: 16-byte aligned
  for (int i = threadIdx.x % 32; i < E / 8; i += 32) q[i] = make_uint4(0u, 0u, 0u, 0u);
  if constexpr (SPLIT)
    for (int i = threadIdx.x % 32; i < E / 8; i += 32) q[3 * E / 8 + i] = make_uint4(0u, 0u, 0u, 0u);
}

// MSA Transformer embedding prologue (/root/reference/esm/model/msa_transformer.py:155-172): for every token of an
// alignment row,  x = LayerNorm(embed_tokens[tok] + embed_positions[pos] + msa_position_embedding[r]) * (1 - is_pad),
// pos = (number of non-pad tokens up to and including this one) + padding_idx for non-pad tokens, padding_idx for pads
// (LearnedPositionalEmbedding.forward, /root/reference/esm/modules.py:241-257).  One block per alignment row.
template <int MAXV>
__global__ void __launch_bounds__(256)
msa_embed_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ embed_table,
                 const float* __restrict__ pos_table, const float* __restrict__ msa_pos, int msa_dim,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ x,
                 int R, int C, int E, int padding_idx) {
  extern __shared__ int s_pos[];  // [C]
  const int row = blockIdx.x;     // b * R + r
  const int r = row % R;
  const int64_t* tok = tokens + (size_t)row * C;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (warp == 0) {
    int base = 0;
    for (int c0 = 0; c0 < C; c0 += 32) {
      const int c = c0 + lane;
      const bool nonpad = c < C && tok[c] != padding_idx;
      const uint32_t bits = __ballot_sync(0xffffffffu, nonpad);
      if (c < C) s_pos[c] = nonpad ? base + __popc(bits & (0xffffffffu >> (31 - lane))) + padding_idx : padding_idx;
      base += __popc(bits);
    }
  }
  __syncthreads();
  const int nvec = E / 4;
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  const float4* m4 = (msa_pos && msa_dim == E) ? reinterpret_cast<const float4*>(msa_pos + (size_t)r * E) : nullptr;
  const float m1 = (msa_pos && msa_dim == 1) ? msa_pos[r] : 0.f;
  for (int c = warp; c < C; c += blockDim.x / 32) {
    const int64_t t = tok[c];
    const float4* e4 = reinterpret_cast<const float4*>(embed_table + (size_t)t * E);
    const float4* p4 = reinterpret_cast<const float4*>(pos_table + (size_t)s_pos[c] * E);
    float4 v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nvec) {
        const float4 a = __ldg(e4 + idx), b = __ldg(p4 + idx);
        float4 o = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        if (m4) {
          const float4 m = __ldg(m4 + idx);
          o.x += m.x; o.y += m.y; o.z += m.z; o.w += m.w;
        } else if (msa_pos) {
          o.x += m1; o.y += m1; o.z += m1; o.w += m1;
        }
        v[i] = o;
        s += (o.x + o.y) + (o.z + o.w);
      }
    }
    const float mean = warp_sum(s) / (float)E;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nvec) {
        const float a = v[i].x - mean, b = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b * b) + (cc * cc + d * d);
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)E + eps);
    const float keep = t == padding_idx ? 0.f : 1.f;
    float4* out = reinterpret_cast<float4*>(x + ((size_t)row * C + c) * E);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nvec) {
        const float4 g = __ldg(g4 + idx), b = __ldg(b4 + idx);
        float4 o;
        o.x = ((v[i].x - mean) * rstd * g.x + b.x) * keep;
        o.y = ((v[i].y - mean) * rstd * g.y + b.y) * keep;
        o.z = ((v[i].z - mean) * rstd * g.z + b.z) * keep;
        o.w = ((v[i].w - mean) * rstd * g.w + b.w) * keep;
        out[idx] = o;
      }
    }
  }
}

// ESM-1b / ESM-1v embedding prologue (/root/reference/esm/model/esm1.py:121-139) in one pass over the rows:
//   x = embed_tokens[tok]; token_dropout: <mask> rows zeroed, x = (x * 0.88) / (1 - n_mask / n_nonpad);
//   x += embed_positions[pos] with pos = cumsum(tok != pad) * (tok != pad) + padding_idx (modules.py:247-248);
//   x = LayerNorm(x) when emb_layer_norm_before is present (gamma != NULL); x *= (1 - is_pad).
// grid (row chunks, B), 8 warps: warp 0 walks the sequence up to the end of the block's chunk with 32-token ballots and
// leaves the chunk's positions in shared memory (any pad pattern, not only trailing pads); with token_dropout every
// thread also counts <mask> / <pad> over the whole sequence.  Then one warp per row, the row held in registers.
template <int MAXV>
__global__ void __launch_bounds__(256)
esm1b_embed_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ embed_table,
                   const float* __restrict__ pos_table, const float* __restrict__ gamma,
                   const float* __restrict__ beta, float eps, int token_dropout, int padding_idx, int mask_idx,
                   float* __restrict__ x, int T, int E) {
  extern __shared__ int s_pos[];  // [rows of this chunk]
  __shared__ int s_cnt[2];
  const int b = blockIdx.y;
  const int64_t* tok = tokens + (size_t)b * T;
  const int rows = (T + gridDim.x - 1) / gridDim.x;
  const int t0 = blockIdx.x * rows, t1 = min(T, t0 + rows);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  if (warp == 0) {
    int base = 0;
    for (int c0 = 0; c0 < t1; c0 += 32) {
      const int c = c0 + lane;
      const bool nonpad = c < T && tok[c] != padding_idx;
      const uint32_t bits = __ballot_sync(0xffffffffu, nonpad);
      if (c >= t0 && c < t1)
        s_pos[c - t0] = nonpad ? base + __popc(bits & (0xffffffffu >> (31 - lane))) + padding_idx : padding_idx;
      base += __popc(bits);
    }
  }
  if (token_dropout) {
    int n_mask = 0, n_pad = 0;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
      const int64_t v = tok[t];
      n_mask += (v == mask_idx);
      n_pad += (v == padding_idx);
    }
    n_mask = __reduce_add_sync(0xffffffffu, n_mask);
    n_pad = __reduce_add_sync(0xffffffffu, n_pad);
    if (lane == 0) {
      atomicAdd(&s_cnt[0], n_mask);
      atomicAdd(&s_cnt[1], n_pad);
    }
  }
  __syncthreads();
  // esm1.py:128-131 (python evaluates 1 - 0.15*0.8 in double, the tensor ops run in fp32: multiply first, then divide)
  const float keep_scale = (float)(1.0 - 0.15 * 0.8);
  const float denom = 1.0f - (float)s_cnt[0] / (float)(T - s_cnt[1]);
  const int nvec = E / 4;
  for (int t = t0 + warp; t < t1; t += blockDim.x / 32) {
    const int64_t v = tok[t];
    const bool zero_emb = token_dropout && v == mask_idx;
    const float4* e4 = reinterpret_cast<const float4*>(embed_table + (size_t)v * E);
    const float4* p4 = reinterpret_cast<const float4*>(pos_table + (size_t)s_pos[t - t0] * E);
    float4 r[MAXV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nvec) {
        float4 e = zero_emb ? make_float4(0.f, 0.f, 0.f, 0.f) : __ldg(e4 + idx);
        if (token_dropout) {
          e.x = (e.x * keep_scale) / denom;
          e.y = (e.y * keep_scale) / denom;
          e.z = (e.z * keep_scale) / denom;
          e.w = (e.w * keep_scale) / denom;
        }
        const float4 p = __ldg(p4 + idx);
        r[i] = make_float4(e.x + p.x, e.y + p.y, e.z + p.z, e.w + p.w);
        s += (r[i].x + r[i].y) + (r[i].z + r[i].w);
      }
    }
    const float keep = v == padding_idx ? 0.f : 1.f;
    float4* out = reinterpret_cast<float4*>(x + ((size_t)b * T + t) * E);
    if (gamma) {  // emb_layer_norm_before (esm1.py:136-137)
      const float mean = warp_sum(s) / (float)E;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int idx = lane + i * 32;
        if (idx < nvec) {
          const float a = r[i].x - mean, bb = r[i].y - mean, cc = r[i].z - mean, d = r[i].w - mean;
          q += (a * a + bb * bb) + (cc * cc + d * d);
        }
      }
      const float rstd = rsqrtf(warp_sum(q) / (float)E + eps);
      const float4* g4 = reinterpret_cast<const float4*>(gamma);
      const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int idx = lane + i * 32;
        if (idx < nvec) {
          const float4 g = __ldg(g4 + idx), bt = __ldg(b4 + idx);
          r[i].x = (r[i].x - mean) * rstd * g.x + bt.x;
          r[i].y = (r[i].y - mean) * rstd * g.y + bt.y;
          r[i].z = (r[i].z - mean) * rstd * g.z + bt.z;
          r[i].w = (r[i].w - mean) * rstd * g.w + bt.w;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nvec) out[idx] = make_float4(r[i].x * keep, r[i].y * keep, r[i].z * keep, r[i].w * keep);
    }
  }
}

// Contact head, per-layer accumulation (/root/reference/esm/modules.py:338-357 with symmetrize :27-29 and apc :32-41,
// restated so that the [B, L*H, S, S] temporaries are never formed): with A_c the eos-masked, bos/eos-cropped attention
// map of channel c = (layer, head),
//     logit_ij = sum_c w_c (A_c + A_c^T)_ij - sum_c (w_c / a12_c) a1_c[i] a1_c[j] + b,
//     a1_c = rowsum(A_c) + colsum(A_c),  a12_c = sum_i a1_c[i].
// This kernel reads one layer's maps [B,H,T,T] ONCE and produces  acc[b,i,j] += sum_h w_h A_h[i,j],  the row sums
// row_sum[b,h,i] and per-CTA partial column sums col_part[b,h,tile,j] (tile = 16-row stripe).  CTA = (16 query rows,
// batch element b), 8 warps, two CTAs per SM when S <= 512; a warp owns RPW rows, a lane owns the columns lane + 32 k:
// row sums by warp shuffles, column sums through an [8][S] shared-memory stage summed in a fixed order.  No atomics:
// every output element has exactly one writer and every sum a fixed order, so contacts are bit-reproducible
// (r01 used float atomicAdd for the column sums).
template <int RPW, int MAXC, int MINB>
__global__ void __launch_bounds__(256, MINB)
contact_accumulate_kernel(const float* __restrict__ attn, long long batch_stride, const float* __restrict__ w,
                          const uint8_t* __restrict__ keep, float* __restrict__ acc, float* __restrict__ row_sum,
                          float* __restrict__ col_part, int H, int T, int lo, int S) {
  extern __shared__ float s_col[];  // [8][S]
  const int b = blockIdx.y;
  const int nt = gridDim.x;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int i0 = blockIdx.x * (8 * RPW) + warp * RPW;
  const uint8_t* kp = keep ? keep + (size_t)b * T : nullptr;
  float ac[RPW][MAXC];
#pragma unroll
  for (int r = 0; r < RPW; ++r)
#pragma unroll
    for (int c = 0; c < MAXC; ++c) ac[r][c] = 0.f;
  float kj[MAXC];
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int j = lane + 32 * c;
    kj[c] = (j < S && (!kp || kp[lo + j])) ? 1.f : 0.f;
  }
  float ki[RPW];
#pragma unroll
  for (int r = 0; r < RPW; ++r) ki[r] = (i0 + r < S && (!kp || kp[lo + i0 + r])) ? 1.f : 0.f;

  // software pipeline over the heads: the RPW x MAXC loads of head h+1 are in flight while head h is reduced
  float v[RPW][MAXC];
  auto load_head = [&](int h) {
    const float* base = attn + (size_t)b * batch_stride + (size_t)h * T * T + (size_t)lo * T + lo;
#pragma unroll
    for (int r = 0; r < RPW; ++r) {
      const float* row = base + (size_t)(i0 + r) * T;
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const int j = lane + 32 * c;
        v[r][c] = (ki[r] != 0.f && j < S) ? __ldg(row + j) : 0.f;
      }
    }
  };
  load_head(0);
  for (int h = 0; h < H; ++h) {
    const float wh = __ldg(w + h);
    float colp[MAXC];
    float rs[RPW];
#pragma unroll
    for (int c = 0; c < MAXC; ++c) colp[c] = 0.f;
#pragma unroll
    for (int r = 0; r < RPW; ++r) {
      rs[r] = 0.f;
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const float x = v[r][c] * kj[c];
        ac[r][c] = fmaf(wh, x, ac[r][c]);
        colp[c] += x;
        rs[r] += x;
      }
    }
    if (h + 1 < H) load_head(h + 1);
#pragma unroll
    for (int r = 0; r < RPW; ++r) {
      const float t = warp_sum(rs[r]);
      if (lane == 0 && i0 + r < S) row_sum[((size_t)b * H + h) * S + i0 + r] = t;
    }
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      const int j = lane + 32 * c;
      if (j < S) s_col[warp * S + j] = colp[c];
    }
    __syncthreads();
    float* cp = col_part + (((size_t)b * H + h) * nt + blockIdx.x) * S;
    for (int j = threadIdx.x; j < S; j += 256) {
      float t = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) t += s_col[q * S + j];
      cp[j] = t;
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < RPW; ++r) {
    if (i0 + r < S) {
      float* dst = acc + ((size_t)b * S + i0 + r) * S;
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const int j = lane + 32 * c;
        if (j < S) dst[j] += ac[r][c];
      }
    }
  }
}

// Contact head tail (modules.py:33-41,352-357): contacts[b,i,j] = sigmoid(acc[b,i,j] + acc[b,j,i]
//   - sum_c u[b,c,i] * a1[b,c,j] + bias),  u = a1 * (w_c / a12_c): the rank-(L*H) APC correction as a 64x64-tiled fp32
// SIMT product (K = L*H channels, 0.75 GFLOP per 510-residue sequence: too small for the tensor path and needs fp32
// operands — the correction cancels most of acc), fused with the symmetrisation, bias and sigmoid.  r01 ran this as a
// cuBLAS sgemm einsum plus four elementwise PyTorch passes.
__global__ void __launch_bounds__(256)
contact_finalize_kernel(const float* __restrict__ acc, const float* __restrict__ u, const float* __restrict__ a1,
                        const float* __restrict__ bias_ptr, float* __restrict__ out, int C, int S) {
  const float bias = bias_ptr ? __ldg(bias_ptr) : 0.f;
  __shared__ float su[16][64 + 1], sa[16][64 + 1];
  const int b = blockIdx.z;
  const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;  // 16 x 16 threads, 4 x 4 outputs each (i = ty + 16 a, j = tx + 16 c)
  float r[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) r[a][c] = 0.f;
  const float* ub = u + (size_t)b * C * S;
  const float* ab = a1 + (size_t)b * C * S;
  for (int c0 = 0; c0 < C; c0 += 16) {
    for (int e = threadIdx.x; e < 16 * 64; e += 256) {
      const int cc = e / 64, x = e % 64;
      const bool okc = c0 + cc < C;
      su[cc][x] = (okc && i0 + x < S) ? ub[(size_t)(c0 + cc) * S + i0 + x] : 0.f;
      sa[cc][x] = (okc && j0 + x < S) ? ab[(size_t)(c0 + cc) * S + j0 + x] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int cc = 0; cc < 16; ++cc) {
      float uu[4], aa[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) { uu[a] = su[cc][ty + 16 * a]; aa[a] = sa[cc][tx + 16 * a]; }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) r[a][c] = fmaf(uu[a], aa[c], r[a][c]);
    }
    __syncthreads();
  }
  const float* accb = acc + (size_t)b * S * S;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int i = i0 + ty + 16 * a;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = j0 + tx + 16 * c;
      if (i < S && j < S) {
        const float z = accb[(size_t)i * S + j] + accb[(size_t)j * S + i] - r[a][c] + bias;
        out[((size_t)b * S + i) * S + j] = 1.0f / (1.0f + __expf(-z));
      }
    }
  }
}

}  // namespace esmb200
