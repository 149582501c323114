// esm_b200 — categorical Jacobian contact map (esm_b200/jacobian.py; Zhang, Wayment-Steele, Brixi, Wang, Kern &
// Ovchinnikov, PNAS 2024), the definition in include/esmb200.h at esmb200_jacobian_contacts.
//
// J [L,20,L,20] fp32 (read only) -> C [L,L] fp32, with every sum in fp64 in a fixed order (no atomics: the result is
// bit-reproducible):
//   jacobian_marginals_kernel  pass 1 over J: S_i[a,j,b] = sum_i J, and per 64-wide j tile the partial sums of
//                              S_j[i,a,b] = sum_j J
//   jacobian_finish_kernel     S_j from its tile partials, S[a,b] = sum_j S_i
//   jacobian_norms_kernel      pass 2 over J: per (i,j) the 20 x 20 block X = J - S_i/L - S_j/L + S/L^2 (the centring
//                              along i and j), double-centred over a and b; N[i,j] = ||X||_F, N[i,i] = 0
//   jacobian_apc_sums_kernel   row and column sums of N
//   jacobian_apc_kernel        A = N - r c^T / sum(r), A[i,i] = 0, C = (A + A^T) / 2
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace esmb200 {

constexpr int kJacAA = 20;          // amino acids per substitution axis
constexpr int kJacTileJ = 64;       // pass 1: j values per block (4 per thread)
constexpr int kJacRowsPerStep = 16; // pass 1: i rows staged per shared-memory reduction
constexpr int kJacNormJ = 8;        // pass 2: (i, j) blocks per CTA

// Scratch layout (fp64 arrays, each 256-byte aligned): S_i [20,L,20] | S_j [L,20,20] | S [20,20] |
// tile partials of S_j [ceil(L/64),L,20,20] | N [L,L] | row sums [L] | column sums [L].
struct JacobianScratch {
  double *s_i, *s_j, *s, *part, *n, *row, *col;
  size_t bytes;
};

inline size_t jac_align(size_t v) { return (v + 255) / 256 * 256; }

inline JacobianScratch jacobian_scratch(char* base, int L) {
  const size_t l = (size_t)L, aa2 = (size_t)kJacAA * kJacAA, tiles = (l + kJacTileJ - 1) / kJacTileJ;
  const size_t sizes[7] = {aa2 * l, aa2 * l, aa2, tiles * l * aa2, l * l, l, l};
  double** dst[7];
  JacobianScratch s;
  dst[0] = &s.s_i; dst[1] = &s.s_j; dst[2] = &s.s; dst[3] = &s.part; dst[4] = &s.n; dst[5] = &s.row; dst[6] = &s.col;
  size_t off = 0;
  for (int k = 0; k < 7; ++k) {
    *dst[k] = base ? reinterpret_cast<double*>(base + off) : nullptr;
    off = jac_align(off + sizes[k] * sizeof(double));
  }
  s.bytes = off;
  return s;
}

// Pass 1. Grid (ceil(L/64), 20): block (jt, a) owns columns j in [64 jt, 64 jt + 64) of the rows (i, a), i < L.
// Thread t = g * 20 + b (g < 16) holds j = 64 jt + g + 16 k, k < 4, so each row's 1280 floats are read as four
// coalesced 320-float runs. It sums its columns over i in i order (S_i), and the 16 rows of one step are reduced over
// (g, k) through shared memory in a fixed order into the tile partial of S_j.
__global__ void __launch_bounds__(320)
jacobian_marginals_kernel(const float* __restrict__ jac, int L, double* __restrict__ s_i, double* __restrict__ part) {
  __shared__ double red[kJacRowsPerStep][320];
  const int t = threadIdx.x, g = t / kJacAA, b = t % kJacAA;
  const int jt = blockIdx.x, a = blockIdx.y;
  const int j0 = jt * kJacTileJ;
  const size_t row_len = (size_t)L * kJacAA;
  double col[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i0 = 0; i0 < L; i0 += kJacRowsPerStep) {
#pragma unroll 4
    for (int ii = 0; ii < kJacRowsPerStep; ++ii) {
      const int i = i0 + ii;
      double s = 0.0;
      if (i < L) {
        const float* row = jac + ((size_t)i * kJacAA + a) * row_len + (size_t)j0 * kJacAA;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int j = j0 + g + 16 * k;
          if (j < L) {
            const double v = (double)row[t + 320 * k];
            col[k] += v;
            s += v;
          }
        }
      }
      red[ii][t] = s;
    }
    __syncthreads();
    {  // thread t = ii * 20 + b: row i0 + ii, column b
      const int ii = t / kJacAA, i = i0 + ii;
      if (i < L) {
        double s = 0.0;
        for (int gg = 0; gg < 16; ++gg) s += red[ii][gg * kJacAA + b];
        part[(((size_t)jt * L + i) * kJacAA + a) * kJacAA + b] = s;
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int j = j0 + g + 16 * k;
    if (j < L) s_i[((size_t)a * L + j) * kJacAA + b] = col[k];
  }
}

// S_j[i,a,b] = sum over the j tiles of their partials, in tile order (threads e < 400 L); S[a,b] = sum_j S_i[a,j,b] in
// j order (the next 400 threads).
__global__ void __launch_bounds__(256)
jacobian_finish_kernel(const double* __restrict__ s_i, const double* __restrict__ part, int L, double* __restrict__ s_j,
                       double* __restrict__ s) {
  const size_t n = (size_t)L * kJacAA * kJacAA;
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) {
    const int tiles = (L + kJacTileJ - 1) / kJacTileJ;
    double acc = 0.0;
    for (int jt = 0; jt < tiles; ++jt) acc += part[(size_t)jt * n + e];
    s_j[e] = acc;
  } else if (e < n + kJacAA * kJacAA) {
    const int ab = (int)(e - n), a = ab / kJacAA, b = ab % kJacAA;
    double acc = 0.0;
    for (int j = 0; j < L; ++j) acc += s_i[((size_t)a * L + j) * kJacAA + b];
    s[ab] = acc;
  }
}

// Pass 2. Grid (ceil(L/8), L): block (jt, i) owns the blocks (i, j), j in [8 jt, 8 jt + 8). Thread t = jj * 20 + b
// reads J[i, a, 8 jt + jj, b] for every a (each row (i, a) gives one coalesced 160-float run), centres it along i and j,
// and keeps it in shared memory; the row means over b, the column means over a and the grand mean then double-centre
// the 20 x 20 block, and N[i,j] is the root of its fixed-order sum of squares.
__global__ void __launch_bounds__(kJacNormJ * kJacAA)
jacobian_norms_kernel(const float* __restrict__ jac, const double* __restrict__ s_i, const double* __restrict__ s_j,
                      const double* __restrict__ s, int L, double* __restrict__ n_out) {
  __shared__ double xs[kJacNormJ][kJacAA][kJacAA];
  __shared__ double rmean[kJacNormJ][kJacAA];
  __shared__ double ssq[kJacNormJ][kJacAA];
  const int t = threadIdx.x, jj = t / kJacAA, b = t % kJacAA;
  const int i = blockIdx.y, j = blockIdx.x * kJacNormJ + jj;
  const bool valid = j < L;
  const double inv_l = 1.0 / (double)L, inv_l2 = inv_l * inv_l;
  const size_t row_len = (size_t)L * kJacAA;
  double cm = 0.0;
#pragma unroll 4
  for (int a = 0; a < kJacAA; ++a) {
    double x = 0.0;
    if (valid) {
      x = (double)jac[((size_t)i * kJacAA + a) * row_len + (size_t)j * kJacAA + b] -
          s_i[((size_t)a * L + j) * kJacAA + b] * inv_l - s_j[((size_t)i * kJacAA + a) * kJacAA + b] * inv_l +
          s[a * kJacAA + b] * inv_l2;
    }
    xs[jj][a][b] = x;
    cm += x;
  }
  cm *= 1.0 / kJacAA;
  __syncthreads();
  {  // thread t = jj * 20 + a: the mean of row a over b
    const int a = t % kJacAA;
    double r = 0.0;
    for (int bb = 0; bb < kJacAA; ++bb) r += xs[jj][a][bb];
    rmean[jj][a] = r * (1.0 / kJacAA);
  }
  __syncthreads();
  double gm = 0.0;
  for (int a = 0; a < kJacAA; ++a) gm += rmean[jj][a];
  gm *= 1.0 / kJacAA;
  double q = 0.0;
  for (int a = 0; a < kJacAA; ++a) {
    const double y = xs[jj][a][b] - rmean[jj][a] - cm + gm;
    q = fma(y, y, q);
  }
  ssq[jj][b] = q;
  __syncthreads();
  if (t < kJacNormJ) {
    const int jw = blockIdx.x * kJacNormJ + t;
    if (jw < L) {
      double tot = 0.0;
      for (int bb = 0; bb < kJacAA; ++bb) tot += ssq[t][bb];
      n_out[(size_t)i * L + jw] = jw == i ? 0.0 : sqrt(tot);
    }
  }
}

// Blocks [0, ceil(L/256)): column sums, one thread per column in i order. The rest: row sums, one warp per row (8 per
// block), lane-strided partials joined by a fixed xor-shuffle tree.
__global__ void __launch_bounds__(256)
jacobian_apc_sums_kernel(const double* __restrict__ n, int L, double* __restrict__ row, double* __restrict__ col) {
  const int col_blocks = (L + 255) / 256;
  if ((int)blockIdx.x < col_blocks) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    if (j < L) {
      double acc = 0.0;
      for (int i = 0; i < L; ++i) acc += n[(size_t)i * L + j];
      col[j] = acc;
    }
    return;
  }
  const int i = ((int)blockIdx.x - col_blocks) * 8 + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (i >= L) return;
  double acc = 0.0;
  for (int j = lane; j < L; j += 32) acc += n[(size_t)i * L + j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) row[i] = acc;
}

// Every block first forms the total sum(row) with the same fixed-order reduction, then writes its grid-stride share of
// C[i,j] = (A[i,j] + A[j,i]) / 2, A[i,j] = N[i,j] - row[i] col[j] / total off the diagonal and 0 on it. An all-zero N
// gives 0 / 0 = NaN off the diagonal, as the definition does.
__global__ void __launch_bounds__(256)
jacobian_apc_kernel(const double* __restrict__ n, const double* __restrict__ row, const double* __restrict__ col, int L,
                    float* __restrict__ out) {
  __shared__ double red[256];
  double acc = 0.0;
  for (int i = threadIdx.x; i < L; i += 256) acc += row[i];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  const double total = red[0];
  const size_t count = (size_t)L * L;
  for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < count; e += (size_t)gridDim.x * 256) {
    const int i = (int)(e / L), j = (int)(e % L);
    double c = 0.0;
    if (i != j) {
      const double a_ij = n[(size_t)i * L + j] - row[i] * col[j] / total;
      const double a_ji = n[(size_t)j * L + i] - row[j] * col[i] / total;
      c = (a_ij + a_ji) * 0.5;
    }
    out[e] = (float)c;
  }
}

}  // namespace esmb200
